"""TEST INFRASTRUCTURE: tests/forced_replica.py over several chunks with the KV memory in the graph.  In the one-chunk replica the memory rows
of K / V are constants read from the tape; here they are the previous chunk's forced K / V (its rows t .. t + maxlen of [memory | chunk],
lib/xf.py:366-391), so autograd through a window of chunks is the exact gradient at the CUDA forward's operating point, through the memory.
The replica's own code is reused: its `torch.cat` of [memory | chunk] is given the carried memory, and its latent is taken where the first
head reads it (as in tests/forced_replica_rl.py)."""
import types

import torch
import torch.nn.functional as F

import forced_replica


class _TorchShim:
    """`torch` for the replica, with `cat` replaced."""

    def __init__(self, cat):
        self.cat = cat

    def __getattr__(self, name):
        return getattr(torch, name)


def forced_chunk(sd, cfg, tape, img_u8, first, mem=None, temperature=2.0):
    """One chunk at the taped operating point -> (latent (N, h), state_out [(k, v)] per layer).  `mem`: None (the tape's memory rows as
    constants, the first chunk of a window) or the previous chunk's state_out."""
    B, t = img_u8.shape[:2]
    maxlen = cfg.maxlen
    seen, out, calls = {}, [], [0]

    def linear(x, w, b=None):
        if w is sd["pi_head.camera.linear_layer.weight"]:
            seen["lat"] = x
        return F.linear(x, w, b)

    def cat(parts, dim=0):
        l, which = divmod(calls[0], 2)  # the replica concatenates K then V of each layer, in layer order
        calls[0] += 1
        taped_mem, new = parts
        m = taped_mem if mem is None else forced_replica._sub(mem[l][which], taped_mem)
        full = torch.cat([m, new], dim)
        if which == 0:
            out.append([full[:, t:t + maxlen]])
        else:
            out[l].append(full[:, t:t + maxlen])
        return full

    shim = types.SimpleNamespace(**{k: getattr(F, k) for k in dir(F) if not k.startswith("_")})
    shim.linear = linear
    actions = {n: torch.zeros(B, t, 1, dtype=torch.int64, device=img_u8.device) for n in ("camera", "buttons")}
    saved = forced_replica.F, forced_replica.torch
    forced_replica.F, forced_replica.torch = shim, _TorchShim(cat)
    try:
        forced_replica.forced_loss(sd, cfg, tape, img_u8, first, actions, temperature)
    finally:
        forced_replica.F, forced_replica.torch = saved
    return seen["lat"], [tuple(kv) for kv in out]


def forced_pd(sd, lat, B, t, temperature=2.0):
    pd = {}
    for name in ("camera", "buttons"):
        lin = f"pi_head.{name}.linear_layer"
        pd[name] = F.log_softmax(F.linear(lat, sd[f"{lin}.weight"], sd[f"{lin}.bias"]).float() / temperature, dim=-1).reshape(B, t, 1, -1)
    return pd


def forced_window(sd, cfg, tapes, chunks):
    """pd per chunk of a window: `tapes` the CUDA forward's tape per call, `chunks` (img, first) per call; the first chunk's memory is
    constant (as the caller's detached or initial state is)."""
    mem, pds = None, []
    for tape, (img, first) in zip(tapes, chunks):
        B, t = img.shape[:2]
        lat, mem = forced_chunk(sd, cfg, tape, img, first, mem)
        pds.append(forced_pd(sd, lat, B, t))
    return pds
