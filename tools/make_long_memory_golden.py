#!/usr/bin/env python
"""Generates tests/golden/long_memory.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_long_memory_golden.py

The reference MinecraftAgentPolicy at the SMALL config of tests/common.py with a KV memory longer than the released models' 128 frames,
seeded weights with perturbed norms and biases, for two memory sizes:

    m1920   attention_memory_size 2048, timesteps 128 (maxlen 1920, the reference's default), chunks of T = 128
    m300    attention_memory_size 364, timesteps 64 (maxlen 300, not a multiple of any tile), chunks of T = 64

and per memory size, all at B = 2:

    forward   enough chunks for the memory to fill and wrap, an episode start at the beginning of row 1's tenth (m300: fourth) chunk:
              log-prob samples (camera in full, buttons at oracle/make_golden.COLS) and vpred of the last chunk, the final state
              (mask in full, K / V at the rows of state_rows())
    window    a no_grad warm-up that fills the memory, its state as a leaf, two chunks with the BC loss on both, ONE backward: the loss,
              per parameter the gradient's norm and a fixed element sample, and the state gradient's norms and rows
    chunk     (m1920) one chunk from the warm-up state, detached, the BC loss: what BCTrainer computes
    rl        (m1920) the same chunk with the RL loss of tools/make_rl_golden.py at kl_coef = 0 (no reference policy)
    loop      (m1920) four T = 1 calls from the warm-up state with the loss summed (each / 4), ONE backward"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402
from make_autograd_golden import _grads  # noqa: E402
from make_bptt_golden import bc_loss, leaf_state  # noqa: E402

WSEED = 5
B = 2
LOOP_CALLS = 4
VF_COEF, CLIP = 0.5, 0.2
RATIOS = (0.5, 0.7, 0.9, 1.0, 1.1, 1.35, 1.6, 0.75)
CONFIGS = {  # name: (attention_memory_size, timesteps, forward chunks, chunk index of the episode start, warm-up chunks)
    "m1920": (2048, 128, 17, 9, 15),
    "m300": (364, 64, 7, 3, 5),
}


def policy_kwargs(name):
    from common import small_kwargs

    ams, T = CONFIGS[name][:2]
    return small_kwargs(timesteps=T, attention_memory_size=ams)


def state_rows(maxlen):
    return torch.cat([torch.arange(0, maxlen, 241), torch.tensor([maxlen - 1])])


def _chunk(g, T, reset=None):
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    if reset is not None:
        first[reset] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    return img, first, actions


def forward_inputs(name):
    _, T, n, reset_at, _ = CONFIGS[name]
    g = torch.Generator().manual_seed(51)
    return [_chunk(g, T, reset=(1, 0) if c == reset_at else None) for c in range(n)]


def warmup_inputs(name):
    _, T, _, _, n = CONFIGS[name]
    g = torch.Generator().manual_seed(52)
    return [_chunk(g, T) for _ in range(n)]


def window_inputs(name):
    T = CONFIGS[name][1]
    g = torch.Generator().manual_seed(53)
    return [_chunk(g, T, reset=(0, 0) if c == 1 else None) for c in range(2)]


def chunk_inputs(name):
    """one chunk plus the RL inputs (advantages, returns, the ratio of each frame to its old log-prob)"""
    T = CONFIGS[name][1]
    g = torch.Generator().manual_seed(54)
    img, first, actions = _chunk(g, T)
    signs = torch.tensor((1.0, -1.0, 1.0, -1.0, -1.0, 1.0, -1.0, -1.0))
    adv = signs.repeat(B * T // len(signs)).reshape(B, T) * (0.5 + torch.rand(B, T, generator=g))
    returns = 3.0 + 2.0 * torch.randn(B, T, generator=g)
    ratios = torch.tensor(RATIOS).repeat(B * T // len(RATIOS)).reshape(B, T)
    return img, first, actions, adv, returns, ratios


def loop_inputs(name):
    g = torch.Generator().manual_seed(55)
    return [_chunk(g, 1) for _ in range(LOOP_CALLS)]


def pd_sample(pd):
    return dict(camera=pd["camera"].detach().clone(), buttons=pd["buttons"].detach()[..., MG.COLS].clone())


def state_sample(st, maxlen):
    rows = state_rows(maxlen)
    return [(m.clone(), k.detach()[:, rows].clone(), v.detach()[:, rows].clone()) for m, (k, v) in st]


def state_grad_sample(st, maxlen):
    rows = state_rows(maxlen)
    return [dict(norm=torch.stack([k.grad.norm(), v.grad.norm()]), k=k.grad[:, rows].clone(), v=v.grad[:, rows].clone()) for _, (k, v) in st]


def warm_state(pol, name):
    st = pol.initial_state(B)
    with torch.no_grad():
        for img, first, _ in warmup_inputs(name):
            _, st = pol({"img": img}, first, st)
    return st


def make_case(name):
    pkw = policy_kwargs(name)
    maxlen = CONFIGS[name][0] - CONFIGS[name][1]
    out = dict(policy_kwargs=pkw)
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    out["schema"] = MG.schema_of(pol.state_dict())
    # -- forward
    st, rec = pol.initial_state(B), []
    with torch.no_grad():
        for img, first, _ in forward_inputs(name):
            (pd, v, _), st = pol({"img": img}, first, st)
            rec.append((pd, v))
    out["forward"] = dict(chunks=[dict(pd=pd_sample(pd), vpred=v.clone()) for pd, v in rec[-1:]], state=state_sample(st, maxlen))
    warm = warm_state(pol, name)
    # -- a two-chunk window from a leaf state, ONE backward
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    st = leaf_state(warm)
    s, loss = st, 0.0
    for img, first, actions in window_inputs(name):
        (pd, _, _), s = pol({"img": img}, first, s)
        loss = loss + bc_loss(pd, actions)
    loss.backward()
    out["window"] = dict(loss=loss.detach().clone(), grads=_grads(pol), state_grad=state_grad_sample(st, maxlen))
    if name != "m1920":
        return out
    # -- one chunk from the detached warm-up state: the BC loss, then the RL loss at kl_coef = 0
    img, first, actions, adv, returns, ratios = chunk_inputs(name)
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    (pd, _, _), _ = pol({"img": img}, first, warm)
    loss = bc_loss(pd, actions)
    loss.backward()
    out["chunk"] = dict(loss=loss.detach().clone(), grads=_grads(pol))
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    pol.train()
    T = img.shape[1]
    N = B * T
    flat = lambda pd: {k: v.reshape(N, 1, *v.shape[2:]) for k, v in pd.items()}  # noqa: E731
    fa = {k: v.reshape(N, 1) for k, v in actions.items()}
    with torch.no_grad():
        (pd0, _, _), _ = pol({"img": img}, first, warm)
        old = pol.get_logprob_of_action(flat(pd0), fa).reshape(B, T) - torch.log(ratios)
    (pd, vpred, _), _ = pol({"img": img}, first, warm)
    ratio = torch.exp(pol.get_logprob_of_action(flat(pd), fa).reshape(B, T) - old)
    l_pi = -torch.min(ratio * adv, ratio.clamp(1 - CLIP, 1 + CLIP) * adv).mean()
    loss = l_pi + VF_COEF * pol.value_head.loss(vpred, returns[..., None])
    loss.backward()
    out["rl"] = dict(loss=loss.detach().clone(), grads=_grads(pol), old_logprob=old.clone())
    # -- four one-frame calls, one backward
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    st, loss = [(m, (k.clone(), v.clone())) for m, (k, v) in warm], 0.0
    for img, first, actions in loop_inputs(name):
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss + bc_loss(pd, actions) / LOOP_CALLS
    loss.backward()
    out["loop"] = dict(loss=loss.detach().clone(), grads=_grads(pol))
    return out


def make_long_memory():
    """The fixture as a dict (also called by tests/test_long_memory_golden.py for the live comparison)."""
    return dict(wseed=WSEED, perturbed=True, **{name: make_case(name) for name in CONFIGS})


if __name__ == "__main__":
    MG._save("long_memory", make_long_memory())
