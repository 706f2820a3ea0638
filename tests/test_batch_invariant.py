"""The batch-invariant mode's host logic on the CPU, through the test-only emulation of the ops (tests/emu_invariant_ops.py): which ops a
step in the mode calls and with which plan, the per-environment sampling counter `RingState.steps` for whole-ring steps, views and inert
rows, `noise_keys`, the graph keys, every refusal (raised before any op), and the numpy Philox4x32-10 that the keyed sampling is checked
against.  tests/test_gpu_batch_invariant.py checks the guarantee itself on the kernels."""
import numpy as np
import pytest
import torch

import emu_invariant_ops
from common import make_policy, small_kwargs
from test_autograd import emulated  # noqa: F401  (fixture)
from test_ring_rows import rows_emu  # noqa: F401  (fixture)
from test_ring_state import random_state
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import GraphedAct, RingState

E = 5
NEW_OPS = ("gemm_rowwise", "conv3x3_zp_plan", "maxpool3s2_plan", "attention_plan", "attention_ring_plan", "ring_noise_keys", "gumbel_argmax_keyed")
ONE_ROW = {"gemm": "gemm_rowwise", "conv3x3_zp": "conv3x3_zp_plan", "maxpool3s2": "maxpool3s2_plan", "attention": "attention_plan",
           "gumbel_argmax": "gumbel_argmax_keyed"}


class Recorder:
    """Records (name, kwargs) of every op called through `ops`."""

    def __init__(self, monkeypatch):
        self.calls = []
        for name in dir(ops):
            fn = getattr(ops, name)
            if not name.startswith("_") and callable(fn) and getattr(fn, "__module__", "").startswith("emu_"):
                monkeypatch.setattr(ops, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        def run(*args, **kwargs):
            self.calls.append((name, kwargs))
            return fn(*args, **kwargs)
        return run


@pytest.fixture()
def inv_emu(rows_emu, monkeypatch):  # noqa: F811
    for name in NEW_OPS:
        monkeypatch.setattr(ops, name, getattr(emu_invariant_ops, name))
    yield


def _step(B, g):
    return {"img": torch.randint(0, 256, (B, 32, 32, 3), dtype=torch.uint8, generator=g)}, torch.rand(B, generator=g) < 0.2


# -- the numpy Philox ------------------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """The known-answer vectors of the Random123 distribution for philox4x32-10."""
    f = emu_invariant_ops.philox4x32_10
    assert f([0, 0, 0, 0], [0, 0]).tolist() == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert f([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2).tolist() == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert f([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0]).tolist() == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_keyed_uniforms_stay_inside_the_unit_interval():
    """The extreme Philox words give uniforms strictly inside (0, 1) in fp32: a uniform of 1 would make its column's score +inf.  Seed 0,
    head 1, stream 0, step 881 draws the word 0xffffffdc for column 8114 of the buttons head."""
    x = np.array([0, 1, 511, 512, 0xFFFFFE00, 0xFFFFFF00, 0xFFFFFFDC, 0xFFFFFFFF], dtype=np.uint64)
    u = ((x >> np.uint64(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    assert (u > 0).all() and (u < 1).all() and np.isfinite(np.log(-np.log(u))).all()
    assert int(emu_invariant_ops.philox4x32_10([8114 // 4, 1, 0, 881], [0, 0])[8114 % 4]) == 0xFFFFFFDC
    lg = torch.full((1, 8641), -10.0)
    lg[0, 8114], lg[0, 3] = -1e4, 50.0
    keys = torch.tensor([[0, 881]])
    assert np.isfinite(emu_invariant_ops.keyed_scores(lg, keys, 0, 1)).all()
    assert int(emu_invariant_ops.gumbel_argmax_keyed(lg, keys, 0, 1)[0]) == 3


def test_keyed_uniforms_properties():
    keys = np.array([[3, 7], [3, 7], [3, 8], [4, 7]])
    u = emu_invariant_ops.keyed_uniforms(keys, 5, 1, 1000)
    assert u.dtype == np.float32 and (u > 0).all() and (u < 1).all()
    assert np.array_equal(u[0], u[1])  # the same (seed, stream, step): the same noise in any row
    assert not np.array_equal(u[0], u[2]) and not np.array_equal(u[0], u[3])  # another step, another stream
    assert not np.array_equal(u[0], emu_invariant_ops.keyed_uniforms(keys, 6, 1, 1000)[0])  # another seed
    assert not np.array_equal(u[0], emu_invariant_ops.keyed_uniforms(keys, 5, 0, 1000)[0])  # another head
    assert abs(float(u.mean()) - 0.5) < 0.02
    big = emu_invariant_ops.keyed_uniforms(np.array([[0, 0]]), 2 ** 40 + 3, 0, 8)  # the seed's high word is part of the key
    assert not np.array_equal(big, emu_invariant_ops.keyed_uniforms(np.array([[0, 0]]), 3, 0, 8))


# -- which ops run, with which plan -----------------------------------------------------------------------------------------------------
def test_mode_runs_one_row_plans(inv_emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(0)
    obs, first = _step(3, g)
    state = random_state(g, pol, 3)
    rec = Recorder(monkeypatch)
    pol.act(obs, first, state, stochastic=False)
    default = [n for n, _ in rec.calls if n != "require_cuda"]
    assert not set(NEW_OPS) & set(default)
    rec.calls.clear()
    pol.set_batch_invariant(True, seed=4)
    pol.act(obs, first, state, noise_keys=torch.zeros((3, 2), dtype=torch.int64))
    names = [n for n, _ in rec.calls if n != "require_cuda"]
    assert names == [ONE_ROW.get(n, n) for n in default]  # the same ops in the same order, each with the one-row plan
    assert all(kw.get("plan_frames", 1) == 1 and kw.get("plan_batch", 1) == 1 for _, kw in rec.calls)
    assert [n for n, _ in rec.calls].count("gumbel_argmax_keyed") == len(pol.head_specs)
    rec.calls.clear()
    pol.set_batch_invariant(False)
    pol.act(obs, first, state, stochastic=False)
    assert [n for n, _ in rec.calls if n != "require_cuda"] == default  # toggled off: the default calls again


# -- the sampling counter of a ring -----------------------------------------------------------------------------------------------------
def test_ring_steps_counter(inv_emu):
    pol, _, _ = make_policy(small_kwargs())
    pol.set_batch_invariant(True, seed=9)
    g = torch.Generator().manual_seed(1)
    ring = RingState.from_pytree(pol, random_state(g, pol, E))
    assert ring.steps is None
    obs, first = _step(E, g)
    pol.v(obs, first, ring)  # no sampling: no counter
    assert ring.steps is None
    pol.act(obs, first, ring)
    assert ring.steps.tolist() == [1] * E
    idx = [3, -1, 0, -1]
    obs, first = _step(len(idx), g)
    pol.act(obs, first, ring.rows(idx))
    assert ring.steps.tolist() == [2, 1, 1, 2, 1]  # listed rows only, never an inert one
    pol.act(obs, first, ring.rows(idx), stochastic=False)  # a deterministic step is still a step of those environments
    assert ring.steps.tolist() == [3, 1, 1, 3, 1]
    before = ring.steps.clone()
    ring.load_(ring.to_pytree())
    assert torch.equal(ring.steps, before)
    ring.rows([1, 4]).load_(ring.rows([1, 4]).to_pytree())
    assert torch.equal(ring.steps, before)
    pol.set_batch_invariant(False)
    obs, first = _step(E, g)
    pol.act(obs, first, ring)  # the default mode does not touch it
    assert torch.equal(ring.steps, before)


def test_ring_keys_are_environment_and_step(inv_emu, monkeypatch):
    """A ring step samples row b of environment e with key (e, steps[e]); replaying from a set counter draws the same action."""
    pol, _, _ = make_policy(small_kwargs())
    pol.set_batch_invariant(True, seed=2)
    g = torch.Generator().manual_seed(3)
    ring = RingState.from_pytree(pol, random_state(g, pol, E))
    ring._alloc_steps()[:] = torch.tensor([5, 6, 7, 8, 9])
    seen = []
    monkeypatch.setattr(ops, "gumbel_argmax_keyed", lambda lg, keys, seed, head: (seen.append((keys.clone(), seed, head)),
                                                                                    emu_invariant_ops.gumbel_argmax_keyed(lg, keys, seed, head))[1])
    idx = [4, -1, 1]
    obs, first = _step(3, g)
    pol.act(obs, first, ring.rows(idx))
    assert [s[2] for s in seen] == list(range(len(pol.head_specs))) and all(s[1] == 2 for s in seen)
    assert seen[0][0].tolist() == [[4, 9], [-1, 0], [1, 6]]


# -- noise_keys and the refusals -------------------------------------------------------------------------------------------------------
def _raises_before_any_op(monkeypatch, exc, fn, match=None):
    rec = Recorder(monkeypatch)
    with pytest.raises(exc, match=match):
        fn()
    assert rec.calls == [], rec.calls


def test_refusals_before_any_op(inv_emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(4)
    obs, first = _step(2, g)
    state = random_state(g, pol, 2)
    keys = torch.zeros((2, 2), dtype=torch.int64)
    # noise_keys without the mode
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol.act(obs, first, state, noise_keys=keys), "batch-invariant")
    pol.set_batch_invariant(True)
    # a stochastic pytree act without keys; keys of the wrong shape or type; keys for a ring
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol.act(obs, first, state), "noise_keys")
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol.act(obs, first, state, noise_keys=keys[:1]), "noise_keys")
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol.act(obs, first, state, noise_keys=keys.int()), "noise_keys")
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol.act(obs, first, state, noise_keys=keys.t().contiguous().t()), "contiguous")
    ring = RingState.from_pytree(pol, state)
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol.act(obs, first, ring, noise_keys=keys), "RingState.steps")
    # T > 1
    chunk = {"img": torch.zeros((2, 3, 32, 32, 3), dtype=torch.uint8)}
    _raises_before_any_op(monkeypatch, ValueError, lambda: pol(chunk, torch.zeros((2, 3), dtype=torch.bool), state), "one-frame")
    # the fp32-parity mode
    pol.set_precision("fp32")
    _raises_before_any_op(monkeypatch, NotImplementedError, lambda: pol.act(obs, first, state, noise_keys=keys), "bf16")
    pol.set_precision("bf16")
    # what needs no key
    pol.act(obs, first, state, stochastic=False)
    ac, _, _ = pol.act(obs, first, state, stochastic=False)
    pol.act(obs, first, state, taken_action={k: v.clone() for k, v in ac.items()})


def test_pytree_keys_pick_the_action(inv_emu):
    """A pytree act samples row b with noise_keys[b]: the same key and logits in another row and another batch give the same action."""
    pol, _, _ = make_policy(small_kwargs())
    pol.set_batch_invariant(True, seed=11)
    g = torch.Generator().manual_seed(5)
    obs, first = _step(3, g)
    state = random_state(g, pol, 3)
    keys = torch.tensor([[0, 4], [1, 4], [2, 4]])
    ac, _, res = pol.act(obs, first, state, noise_keys=keys, return_pd=True)
    for name, pd in res["pd"].items():
        want = emu_invariant_ops.gumbel_argmax_keyed(pd, keys, 11, list(pol.head_specs).index(name))
        assert torch.equal(ac[name], want)
    # one row alone with its key, in a batch of one
    ac1, _, _ = pol.act({"img": obs["img"][2:]}, first[2:], [(m[2:], (k[2:], v[2:])) for m, (k, v) in state], noise_keys=keys[2:])
    rp = {k: v[2:] for k, v in res["pd"].items()}
    for name in ac1:
        assert torch.equal(ac1[name], emu_invariant_ops.gumbel_argmax_keyed(rp[name], keys[2:], 11, list(pol.head_specs).index(name)))


def test_graph_keys_on_mode_and_seed():
    """GraphedAct keys its graphs on the mode and the seed (and the address of the ring's counter), so toggling either captures again."""
    pol, _, _ = make_policy(small_kwargs())
    ga = GraphedAct.__new__(GraphedAct)
    ga.policy, ga.memory, ga.state = pol, "pytree", None
    k0 = ga._key(True)
    pol.set_batch_invariant(True, seed=1)
    k1 = ga._key(True)
    pol.set_batch_invariant(True, seed=2)
    k2 = ga._key(True)
    pol.set_batch_invariant(False, seed=2)
    assert len({k0, k1, k2}) == 3 and ga._key(True) == k0 and ga._key(False) != k0
    ga.memory, ga.state = "ring", RingState.zeros(pol, 2)
    pol.set_batch_invariant(True)
    before = ga._key(True)
    ga.state._alloc_steps()
    assert ga._key(True) != before
