#!/usr/bin/env python
"""Generates tests/golden/bptt_gradient.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_bptt_golden.py

The reference model backpropagates through its KV memory when the state is not detached (lib/xf.py:366-391 builds the next memory with
cat and slicing); these are its own autograd gradients for three windows at the SMALL config of tests/common.py (maxlen 8, seeded weights
with perturbed norms and biases), the state carried attached and ONE backward per window:

    two_chunks  B = 2, two chunks of T = 8 with an episode start at the beginning of row 1's second chunk, the BC loss on both chunks
    uneven      B = 2, a no_grad warm-up chunk of T = 8 whose state becomes a leaf, then chunks of T = 3, 3, 5 (an episode start on row 0
                of the second), the BC loss on the last chunk only; the gradient wrt the leaf state is stored too
    loop        behavioural_cloning.py's shape, B = 1, T = 1, over six calls, the loss summed (each sample / 6)

Per case: the loss, per parameter the gradient's norm and a fixed element sample (or None), and for `uneven` the state gradient.  No state
dict is stored."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402
from make_autograd_golden import _grads  # noqa: E402

WSEED = 5
LOOP_CALLS = 6


def _chunk(g, B, T, reset=None):
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    if reset is not None:
        first[reset] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    return img, first, actions


def two_chunks_inputs():
    g = torch.Generator().manual_seed(31)
    return [_chunk(g, 2, 8, reset=(1, 0) if c == 1 else None) for c in range(2)]


def uneven_inputs():
    """(warm-up chunk, [the three chunks])"""
    g = torch.Generator().manual_seed(32)
    warm = _chunk(g, 2, 8)
    return warm, [_chunk(g, 2, t, reset=(0, 0) if c == 1 else None) for c, t in enumerate((3, 3, 5))]


def loop_inputs():
    g = torch.Generator().manual_seed(33)
    return [_chunk(g, 1, 1) for _ in range(LOOP_CALLS)]


def leaf_state(st):
    return [(m, (k.detach().clone().requires_grad_(True), v.detach().clone().requires_grad_(True))) for m, (k, v) in st]


def bc_loss(pd, actions):
    """-mean over the frames of the summed log-probabilities of the demonstrated actions, as a plain gather over the last axis of pd, so
    that the reference's pd and this project's give the same loss whatever their leading shapes."""
    n = actions["camera"].numel()
    return -sum(pd[k].reshape(n, -1).gather(-1, actions[k].reshape(n, 1)).sum() for k in ("camera", "buttons")) / n


def make_bptt_gradient():
    """The fixture as a dict (also called by tests/test_bptt_golden.py for the live comparison)."""
    from common import small_kwargs

    pkw = small_kwargs()
    out = dict(policy_kwargs=pkw, wseed=WSEED, perturbed=True)
    # -- two chunks, the loss on both
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    out["schema"] = MG.schema_of(pol.state_dict())
    st, loss = pol.initial_state(2), 0.0
    for img, first, actions in two_chunks_inputs():
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss + bc_loss(pd, actions)
    loss.backward()
    out["two_chunks"] = dict(loss=loss.detach().clone(), grads=_grads(pol))
    # -- a leaf state, chunks of 3, 3, 5, the loss on the last
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    (img, first, _), chunks = uneven_inputs()
    with torch.no_grad():
        _, st0 = pol({"img": img}, first, pol.initial_state(2))
    st = leaf_state(st0)
    s = st
    for img, first, actions in chunks:
        (pd, _, _), s = pol({"img": img}, first, s)
    loss = bc_loss(pd, actions)
    loss.backward()
    out["uneven"] = dict(loss=loss.detach().clone(), grads=_grads(pol), state_grad=[(k.grad.clone(), v.grad.clone()) for _, (k, v) in st])
    # -- the reference loop's shape, one backward
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    st, loss = pol.initial_state(1), 0.0
    for img, first, actions in loop_inputs():
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss + bc_loss(pd, actions) / LOOP_CALLS
    loss.backward()
    out["loop"] = dict(loss=loss.detach().clone(), grads=_grads(pol))
    return out


if __name__ == "__main__":
    MG._save("bptt_gradient", make_bptt_gradient())
