"""Generates tests/golden/*.pt from the UNMODIFIED reference (run where the reference checkout exists, see oracle/refshim.py):

    python oracle/make_golden.py

Every fixture records what a test that compares with the reference compares against, so that the comparison also runs where the
reference is absent.  Weights are not stored: `seeded_state_dict` fills a state-dict template (the names, shapes and dtypes of the
reference's state dict, stored with each fixture) from a fixed seed, and the inputs come from fixed seeds too; the helpers below
that build weights and inputs are shared by this recipe and the tests.  Large outputs are stored as fixed column samples
(`COLS`), parameter gradients as fixed element samples plus their norms, so that every file stays well under 1 MB.

  tiny_plain / tiny_perturbed        tiny policy, B=3, chunks of 8/8/3/8/1 frames (a reset in chunk 3): logits, vpred, KV state,
                                     masks, sampled actions and their log-prob (`perturbed`: norm affines / biases randomised and q
                                     weights x30, so that layout mistakes that plain init hides show up)
  forward_128px                      one 128x128 frame through the 1x policy (one transformer layer)
  gradient                           the BC loss and its gradient through the reference with autograd, two chunks, KV memory detached
  idm                                a small IDM forward, plus the reference's state-dict schema at the IDM config the CUDA path runs
  codec                              the reference action mapping / action transformer on seeded action batches
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import refshim  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
COLS = torch.randperm(8641, generator=torch.Generator().manual_seed(11))[:128].sort().values  # buttons-head columns kept
TINY = refshim.TINY
IDM_KW = dict(impala_width=1, hidsize=64, attention_heads=2, img_shape=[32, 32, 16],
              conv3d_params=dict(inchan=3, outchan=16, kernel_size=[5, 1, 1], padding=[2, 0, 0]), timesteps=8, attention_memory_size=8)
GRAD_SAMPLES = 32


def seeded_state_dict(template, seed, perturbed=False):
    """Deterministic weights for a state-dict template: matrices ~ N(0, 1/fan_in), norm gains 1 + N(0, 0.1^2) (N(0, 0.1^2) around 1
    also for `perturbed`), biases N(0, 0.01^2) (N(0, 0.1^2) when `perturbed`, which also scales the q projections x30)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(template):
        t = template[k]
        if not t.dtype.is_floating_point:
            out[k] = t.clone()
            continue
        r = torch.randn(t.shape, generator=g, dtype=torch.float32)
        if t.dim() >= 2:
            v = r * (max(t[0].numel(), 1) ** -0.5)
            if perturbed and "q_layer.weight" in k:
                v = v * 30.0
        elif k.endswith("weight"):
            v = 1.0 + 0.1 * r
        else:
            v = (0.1 if perturbed else 0.01) * r
        out[k] = v.to(t.dtype)
    return {k: out[k] for k in template}


def perturb(pol, seed=1):
    """Randomises every norm affine / bias and scales the q weights x30 of a live policy (the live comparisons in tests/test_oracle.py)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in pol.named_parameters():
            if ".norm." in n or n.endswith(".bias") or "_ln." in n or ".n." in n:
                p.add_(torch.randn(p.shape, generator=g) * 0.1)
            if "q_layer.weight" in n:
                p.mul_(30.0)


def schema_of(sd):
    return [(k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()]


def template_from(schema):
    """A state-dict template (zeros of the stored names / shapes / dtypes) for `seeded_state_dict`."""
    return {k: torch.zeros(shape, dtype=getattr(torch, dt)) for k, shape, dt in schema}


def forward_inputs(B=3):
    g = torch.Generator().manual_seed(0)
    chunks = []
    for ci, T in enumerate([8, 8, 3, 8, 1]):
        img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
        first = torch.zeros(B, T, dtype=torch.bool)
        if ci == 3:
            first[1, 0] = True
        chunks.append((img, first))
    return chunks


def img_128px():
    return torch.randint(0, 256, (1, 1, 128, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(3))


def gradient_inputs(B=2, T=8):
    g = torch.Generator().manual_seed(3)
    out = []
    for _ in range(2):
        img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
        actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
        out.append((img, torch.zeros(B, T, dtype=torch.bool), actions))
    return out


def grad_sample_index(name, numel):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    return torch.randperm(numel, generator=g)[:GRAD_SAMPLES]


def idm_img():
    return torch.randint(0, 256, (2, 8, 32, 32, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(4))


def codec_inputs():
    """The seeded action batches of the codec comparison (numpy's PCG64 stream is stable across versions)."""
    rng = np.random.default_rng(0)
    joint = dict(buttons=rng.integers(0, 8641, (500, 1)), camera=rng.integers(0, 121, (500, 1)))
    btn = (rng.random((2000, 20)) < 0.25).astype(np.int64)
    cam = rng.integers(0, 11, (2000, 2))
    cam[rng.random(2000) < 0.4] = 5
    fac = dict(buttons=btn, camera=cam)
    env = {"camera": rng.uniform(-15, 15, (300, 2)), "attack": rng.integers(0, 2, 300), "hotbar.3": rng.integers(0, 2, 300)}
    return joint, fac, env


def _save(name, fx):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".pt")
    torch.save(fx, path)
    print(name, os.path.getsize(path) // 1024, "KiB")


def _ref_policy(pkw, wseed, perturbed=False):
    pol = refshim.make_reference_agent_policy(pkw)
    pol.load_state_dict(seeded_state_dict(pol.state_dict(), wseed, perturbed))
    return pol


def make_forward(pert):
    pkw = refshim.policy_kwargs("2x", **TINY)
    pol = _ref_policy(pkw, 1, pert)
    B = 3
    st = pol.initial_state(B)
    rec = []
    with torch.no_grad():
        for img, first in forward_inputs(B):
            (pd, v, _), st = pol({"img": img}, first, st)
            rec.append(dict(camera=pd["camera"].clone(), buttons=pd["buttons"][..., COLS].clone(), vpred=v.clone(),
                            state=[(s[0].clone(), s[1][0].clone(), s[1][1].clone()) for s in st]))
        torch.manual_seed(7)
        ac = pol.pi_head.sample(pd)
        lp = pol.pi_head.logprob(ac, pd)
    _save("tiny_perturbed" if pert else "tiny_plain",
          dict(policy_kwargs=pkw, schema=schema_of(pol.state_dict()), wseed=1, perturbed=pert, B=B, chunks=rec, sample={k: v.clone() for k, v in ac.items()}, sample_logprob=lp.clone()))


def make_forward_128px():
    pkw = refshim.policy_kwargs("1x", n_recurrence_layers=1)
    pol = _ref_policy(pkw, 2)
    with torch.no_grad():
        (pd, v, _), _ = pol({"img": img_128px()}, torch.zeros(1, 1, dtype=torch.bool), pol.initial_state(1))
    _save("forward_128px", dict(policy_kwargs=pkw, schema=schema_of(pol.state_dict()), wseed=2, camera=pd["camera"].clone(), buttons=pd["buttons"].clone(), vpred=v.clone()))


def make_gradient():
    pkw = refshim.policy_kwargs("2x", **TINY)
    pol = _ref_policy(pkw, 3, perturbed=True)
    pol.train()  # as behavioural_cloning.py leaves it (no dropout / batch-norm in these models: same function)
    B = 2
    st = pol.initial_state(B)
    rec = []
    for img, first, actions in gradient_inputs(B):
        for p in pol.parameters():
            p.grad = None
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = -pol.pi_head.logprob(actions, pd).mean()
        loss.backward()
        st = [(m, (k.detach(), v.detach())) for (m, (k, v)) in st]  # tree_map(lambda x: x.detach(), ...) :111
        grads = {}
        for name, p in pol.named_parameters():
            if p.grad is None:
                grads[name] = None
            else:
                gflat = p.grad.detach().flatten()
                grads[name] = dict(sample=gflat[grad_sample_index(name, gflat.numel())].clone(), norm=gflat.norm().clone())
        rec.append(dict(loss=loss.detach().clone(), grads=grads))
    _save("gradient", dict(policy_kwargs=pkw, schema=schema_of(pol.state_dict()), wseed=3, perturbed=True, B=B, chunks=rec))


def make_idm():
    import vpt_b200

    ns = refshim.load()
    kw = vpt_b200.idm_net_kwargs(**IDM_KW)
    mapper = ns.action_mapping.IDMActionMapping(n_camera_bins=11)
    ref = ns.policy.InverseActionPolicy(action_space=ns.DictType(**mapper.get_action_space_update()), pi_head_kwargs=dict(temperature=2.0),
                                        idm_net_kwargs=kw)
    ref.eval()
    ref.load_state_dict(seeded_state_dict(ref.state_dict(), 4))
    with torch.no_grad():
        (pd, _, _), _ = ref(obs={"img": idm_img()}, first=torch.zeros(2, 8), state_in=ref.initial_state(2))
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
    from test_idm import SMALL_IDM

    ref2 = ns.policy.InverseActionPolicy(action_space=ns.DictType(**mapper.get_action_space_update()), pi_head_kwargs=dict(temperature=2.0),
                                         idm_net_kwargs=vpt_b200.idm_net_kwargs(**SMALL_IDM))
    _save("idm", dict(wseed=4, pd={k: v.clone() for k, v in pd.items()}, schema=schema_of(ref.state_dict()),
                      small_schema=[(k, tuple(v.shape)) for k, v in ref2.state_dict().items()]))


def make_codec():
    ns = refshim.load()
    import lib.actions as ref_actions  # noqa: E402  (importable once refshim.load() has set up sys.path + stubs)
    from video_pre_training_b200 import agent as A

    mapper = ns.action_mapping.CameraHierarchicalMapping(n_camera_bins=11)
    tr = ref_actions.ActionTransformer(**A.ACTION_TRANSFORMER_KWARGS)
    joint, fac, env = codec_inputs()
    fx = dict(n_buttons_joint=len(mapper.BUTTONS_COMBINATIONS),
              idx_to_factored=np.asarray(mapper.BUTTON_IDX_TO_FACTORED).astype(np.uint8),
              idx_camera_off=np.asarray(mapper.BUTTON_IDX_TO_CAMERA_META_OFF).astype(np.uint8),
              to_factored=mapper.to_factored({k: v.copy() for k, v in joint.items()}),
              from_factored=mapper.from_factored({k: v.copy() for k, v in fac.items()}),
              policy2env=tr.policy2env({k: v.copy() for k, v in fac.items()}),
              env2policy=tr.env2policy(env),
              null_buttons_idx=np.asarray(mapper.get_zero_action()["buttons"]), camera_null_idx=int(mapper.camera_null_idx))
    _save("codec", fx)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    make_forward(False)
    make_forward(True)
    make_forward_128px()
    make_gradient()
    make_idm()
    make_codec()
