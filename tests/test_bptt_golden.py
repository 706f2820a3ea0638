"""Truncated BPTT across calls against the reference's own autograd through its KV memory (tests/golden/bptt_gradient.pt, made by
tools/make_bptt_golden.py): two chunks with the loss on both, uneven chunks from a leaf state with the loss on the last (the state
gradient compared too), and the one-frame loop shape with one backward.  Live where the reference checkout is present (the stored fixture
is then also re-derived and compared), against the stored file elsewhere."""
import os
import sys

import torch

import refshim
from test_autograd_golden import _check, _policy
from test_bptt import bptt, emulated, exact  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_bptt_golden as MBG  # noqa: E402

CASES = ("two_chunks", "uneven", "loop")


def _fixture():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "bptt_gradient.pt"), weights_only=False)
    if refshim.available():  # the stored file must still be what the reference computes
        live = MBG.make_bptt_gradient()
        for case in CASES:
            assert abs(live[case]["loss"].item() - fx[case]["loss"].item()) <= 1e-5 * abs(fx[case]["loss"].item()), case
            for n, g in fx[case]["grads"].items():
                lg = live[case]["grads"][n]
                assert (g is None) == (lg is None), (case, n)
                if g is not None:
                    assert (lg["sample"] - g["sample"]).abs().max().item() <= 1e-5 * max(g["norm"].item(), 1e-12), (case, n)
        for (k, v), (lk, lv) in zip(fx["uneven"]["state_grad"], live["uneven"]["state_grad"]):
            assert torch.allclose(lk, k, rtol=1e-5, atol=1e-8 * k.abs().max().item()) and torch.allclose(lv, v, rtol=1e-5, atol=1e-8 * v.abs().max().item())
        fx = live
    return fx


def test_two_chunks_loss_on_both(bptt, exact):  # noqa: F811
    fx = _fixture()
    pol = _policy(fx, fx["wseed"]).set_autograd(True, state_grad=True)
    st, loss = pol.initial_state(2), 0.0
    for img, first, actions in MBG.two_chunks_inputs():
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss + MBG.bc_loss(pd, actions)
    loss.backward()
    assert pol.value_head.linear.weight.grad is None
    assert _check(pol, fx["two_chunks"]["grads"], loss.item(), fx["two_chunks"]["loss"]) > 40


def test_uneven_chunks_and_the_state_gradient(bptt, exact):  # noqa: F811
    fx = _fixture()
    pol = _policy(fx, fx["wseed"]).set_autograd(True, state_grad=True)
    (img, first, _), chunks = MBG.uneven_inputs()
    with torch.no_grad():
        _, st0 = pol({"img": img}, first, pol.initial_state(2))
    st = MBG.leaf_state(st0)
    s = st
    for img, first, actions in chunks:
        (pd, _, _), s = pol({"img": img}, first, s)
    loss = MBG.bc_loss(pd, actions)
    loss.backward()
    assert _check(pol, fx["uneven"]["grads"], loss.item(), fx["uneven"]["loss"]) > 40
    for (_, (k, v)), (gk, gv) in zip(st, fx["uneven"]["state_grad"]):
        for a, b in ((k.grad, gk), (v.grad, gv)):
            assert ((a - b).norm() / b.norm()).item() < 1e-3


def test_one_frame_loop_one_backward(bptt, exact):  # noqa: F811
    fx = _fixture()
    pol = _policy(fx, fx["wseed"]).set_autograd(True, state_grad=True)
    st, loss = pol.initial_state(1), 0.0
    for img, first, actions in MBG.loop_inputs():
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss + MBG.bc_loss(pd, actions) / MBG.LOOP_CALLS
    loss.backward()
    assert _check(pol, fx["loop"]["grads"], loss.item(), fx["loop"]["loss"]) > 40
