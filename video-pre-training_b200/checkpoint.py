"""Checkpoint I/O compatible with the released VPT files (SURVEY section 8 f-4).

    .model    pickle holding the constructor arguments of the policy            run_agent.py:11-14, behavioural_cloning.py:42-47
    .weights  torch.save of MinecraftAgentPolicy.state_dict()                    agent.py:132-135, behavioural_cloning.py:131-132
    training  state_dict + FlatAdamDP state (moments, step count) in one file    (the reference saves weights only)

`resize_memory` adapts a state dict to another KV-memory length (`attention_memory_size - timesteps`).
"""
import pickle

import torch


def load_model_parameters(path_to_model_file):
    """(policy_kwargs, pi_head_kwargs) from a released `.model` file.  The file is a plain nested dict; the reference reads
    ["model"]["args"]["net"]["args"] and ["model"]["args"]["pi_head_opts"] and casts the temperature to float."""
    with open(path_to_model_file, "rb") as fh:
        blob = pickle.load(fh)
    args = blob["model"]["args"]
    policy_kwargs = dict(args["net"]["args"])
    pi_head_kwargs = dict(args["pi_head_opts"])
    pi_head_kwargs["temperature"] = float(pi_head_kwargs["temperature"])
    return policy_kwargs, pi_head_kwargs


def save_weights(policy, path):
    """`th.save(policy.state_dict(), out_weights)` (behavioural_cloning.py:131-132).  Tensors are detached, moved to the CPU and
    made contiguous first: under FlatAdamDP the parameters are views into one flat bucket, which torch.save would otherwise
    serialise as views of a single 2 GB storage."""
    sd = {k: v.detach().to("cpu").contiguous().clone() for k, v in policy.state_dict().items()}
    torch.save(sd, path)


def load_weights(policy, path, map_location=None):
    """agent.py:132-135: `load_state_dict(th.load(path), strict=False)` on the reference schema (identical keys / shapes here).
    In-place copies, so it also works after FlatAdamDP has re-pointed the parameters into its flat bucket."""
    sd = torch.load(path, map_location=map_location or "cpu")
    return policy.load_state_dict(sd, strict=False)


def resize_memory(state_dict, maxlen):
    """A copy of `state_dict` whose relative-position biases (every `...orc_block.b_nd`, shape (nbasis, old maxlen)) are cut or
    zero-padded to (nbasis, maxlen), so that weights trained with one memory length load into a policy built with another
    (`load_state_dict` raises on the shape mismatch otherwise, even with strict=False).  Distance d keeps its column; distances the
    checkpoint never trained get no relative bias.  Every other entry is the same tensor object."""
    maxlen = int(maxlen)
    if maxlen < 0:
        raise ValueError(f"resize_memory: maxlen must be >= 0 (got {maxlen})")
    out = dict(state_dict)
    for k, v in state_dict.items():
        if k.endswith("orc_block.b_nd"):
            if v.dim() != 2:
                raise ValueError(f"resize_memory: {k} has shape {tuple(v.shape)}, expected (nbasis, maxlen)")
            w = v.new_zeros((v.shape[0], maxlen))
            n = min(maxlen, v.shape[1])
            w[:, :n] = v[:, :n]
            out[k] = w
    return out


def save_training_state(path, policy, optimizer):
    """Weights + optimizer moments + step count, to resume a BC run exactly."""
    torch.save({"weights": {k: v.detach().to("cpu").contiguous().clone() for k, v in policy.state_dict().items()},
                "optimizer": optimizer.state_dict()}, path)


def load_training_state(path, policy, optimizer):
    blob = torch.load(path, map_location="cpu")
    policy.load_state_dict(blob["weights"], strict=False)
    optimizer.load_state_dict(blob["optimizer"])
