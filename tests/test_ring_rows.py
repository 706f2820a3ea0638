"""Asynchronous rollouts on the CPU through the test-only torch emulation of the ops (tests/emu_ring_rows_ops.py for the ring kernels with
row maps and per-environment offsets): a step of any subset of a `RingState`'s environments, through `ring.rows(idx)`, is the pytree
forward of those environments' states gathered into a batch, bit for bit, and leaves every other environment's bytes alone.  Also the
round trips of `RingRows.load_` / `to_pytree` and of a ring with per-row offsets, and every call a view cannot serve raising before any
op.  tests/test_gpu_ring_rows.py repeats the schedule through the CUDA kernels at 2x width."""
import pytest
import torch

import emu_ring_ops
import emu_ring_rows_ops
from common import make_policy, small_kwargs
from test_autograd import emulated  # noqa: F401  (fixture)
from test_latents import OpRecorder
from test_ring_state import assert_same_state, random_state
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import GraphedAct, RingRows, RingState
from video_pre_training_b200.training import BCTrainer

E = 5


@pytest.fixture()
def rows_emu(emulated, monkeypatch):  # noqa: F811
    monkeypatch.setattr(ops, "ring_advance", emu_ring_ops.ring_advance)
    for name in ("ring_write", "attention_ring", "ring_advance_rows"):
        monkeypatch.setattr(ops, name, getattr(emu_ring_rows_ops, name))
    yield


class EnvStates:
    """The reference: one reference-format state per environment, as rows (mask (maxlen,), K, V fp32 (maxlen, h)) per layer."""

    def __init__(self, pytree):
        self.env = [[(_mask_rows(m, K.shape[0], K.shape[1])[e], K[e].clone(), V[e].clone()) for m, (K, V) in pytree]
                    for e in range(pytree[0][1][0].shape[0])]
        self.blank = [(torch.zeros_like(m), torch.zeros_like(K), torch.zeros_like(V)) for m, K, V in self.env[0]]  # initial_state

    def gather(self, idx):
        rows = [self.env[e] if e >= 0 else self.blank for e in idx]
        return [(torch.stack([r[l][0] for r in rows])[:, None], (torch.stack([r[l][1] for r in rows]), torch.stack([r[l][2] for r in rows])))
                for l in range(len(self.blank))]

    def scatter(self, idx, pytree):
        for i, e in enumerate(idx):
            if e >= 0:
                self.env[e] = [(_mask_rows(m, K.shape[0], K.shape[1])[i], K[i].clone(), V[i].clone()) for m, (K, V) in pytree]


def _mask_rows(m, B, maxlen):
    return torch.zeros(B, maxlen, dtype=torch.bool) if m is None else m.reshape(B, maxlen)


def _outputs(ac, res, live):
    return ({k: v[live] for k, v in ac.items()}, res["log_prob"][live], res["vpred"][live], {k: v[live] for k, v in res["pd"].items()})


def _same_outputs(a, b):
    (ac0, lp0, v0, pd0), (ac1, lp1, v1, pd1) = a, b
    assert ac0.keys() == ac1.keys() and all(torch.equal(ac0[k], ac1[k]) for k in ac0)
    assert torch.equal(lp0, lp1) and torch.equal(v0, v1)
    assert pd0.keys() == pd1.keys() and all(torch.equal(pd0[k], pd1[k]) for k in pd0)


def _bytes(ring, e):
    return ([k[e].clone() for k in ring.k], [v[e].clone() for v in ring.v], [m[e].clone() for m in ring.mask],
            0 if ring.row_off is None else int(ring.row_off[e]))  # (None: every offset 0; the first view step allocates the zeros)


def _same_bytes(a, b):
    assert all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(a[0] + a[1] + a[2], b[0] + b[1] + b[2]))
    assert a[3] == b[3]


def schedule(g, steps):
    """Per step the environments stepped, in call order: None for a whole-ring step, else a list with -1 for inert padding rows."""
    out = []
    for s in range(steps):
        kind = s % 6
        if kind == 0:
            out.append(None)  # whole ring
        elif kind == 1:
            out.append([int(torch.randint(0, E, (1,), generator=g))])  # a singleton
        elif kind == 2:
            out.append(torch.randperm(E, generator=g).tolist())  # all E, permuted
        else:
            k = int(torch.randint(1, E, (1,), generator=g))
            sub = torch.randperm(E, generator=g)[:k].tolist()
            pad = int(torch.randint(0, 3, (1,), generator=g))
            for _ in range(pad):  # inert rows anywhere in the call
                sub.insert(int(torch.randint(0, len(sub) + 1, (1,), generator=g)), -1)
            out.append(sub)
    return out


def test_async_schedule_is_the_gathered_pytree_forward(rows_emu):
    """E = 5 environments at maxlen 8 over 72 steps: whole-ring steps (which wrap `off`) interleaved with singletons, all E in permuted
    order and subsets padded with -1 (after which every `row_off` has wrapped), with episode resets."""
    pol, _, _ = make_policy(small_kwargs())
    maxlen = pol.net.cfg.maxlen
    assert maxlen == 8
    g = torch.Generator().manual_seed(11)
    start = random_state(g, pol, E)
    ref = EnvStates(start)
    ring = RingState.from_pytree(pol, start)
    whole, stepped = 0, [0] * E
    for s, idx in enumerate(schedule(g, 72)):
        envs = list(range(E)) if idx is None else idx
        B = len(envs)
        live = [i for i, e in enumerate(envs) if e >= 0]
        frames = torch.randint(0, 256, (B, 32, 32, 3), dtype=torch.uint8, generator=g)
        first = torch.rand(B, generator=g) < 0.1
        for i, e in enumerate(envs):
            if e < 0:
                frames[i] = 0
                first[i] = False
        torch.manual_seed(500 + s)
        ac, st, res = pol.act({"img": frames}, first, ref.gather(envs), return_pd=True)
        ref.scatter(envs, st)
        want = _outputs(ac, res, live)
        untouched = [e for e in range(E) if e not in envs]
        before = {e: _bytes(ring, e) for e in untouched}
        state = ring if idx is None else ring.rows(idx)
        torch.manual_seed(500 + s)
        ac, out, res = pol.act({"img": frames}, first, state, return_pd=True)
        assert out is state
        _same_outputs(want, _outputs(ac, res, live))
        assert all(torch.isfinite(res["log_prob"]))  # inert rows too
        for e in untouched:
            _same_bytes(before[e], _bytes(ring, e))
        real = [e for e in envs if e >= 0]
        assert_same_state(ring.rows(real).to_pytree(), ref.gather(real))
        if idx is None:
            whole += 1
        else:
            for e in real:
                stepped[e] += 1
    assert whole > maxlen and min(stepped) > maxlen  # `off` and every `row_off` wrapped
    assert_same_state(ring.to_pytree(), ref.gather(list(range(E))))


def test_view_round_trips(rows_emu):
    pol, _, _ = make_policy(small_kwargs())
    maxlen = pol.net.cfg.maxlen
    g = torch.Generator().manual_seed(12)
    ring = RingState.from_pytree(pol, random_state(g, pol, E))
    assert ring.row_off is None
    for s in range(3):  # `off` at 3
        pol.act({"img": torch.randint(0, 256, (E, 32, 32, 3), dtype=torch.uint8, generator=g)}, torch.zeros(E, dtype=torch.bool), ring)
    view = ring.rows(torch.tensor([4, 1]))
    assert ring.row_off is None  # a view alone allocates nothing
    new = random_state(g, pol, 2)
    before = {e: _bytes(ring, e) for e in (0, 2, 3)}
    everything = ring.to_pytree()
    assert view.load_(new) is view
    assert ring.row_off is not None and int(ring.off) == 3
    assert ring.row_off[[4, 1]].tolist() == [(maxlen - 3) % maxlen] * 2
    assert_same_state(view.to_pytree(), new)
    assert_same_state(ring.rows([1, 4]).to_pytree(), [(m[[1, 0]], (K[[1, 0]], V[[1, 0]])) for m, (K, V) in new])
    for e in (0, 2, 3):
        _same_bytes(before[e], _bytes(ring, e))
    expect = [(m.clone(), (K.clone(), V.clone())) for m, (K, V) in everything]
    for (m, (K, V)), (mn, (Kn, Vn)) in zip(expect, new):
        m[[4, 1]], K[[4, 1]], V[[4, 1]] = mn, Kn, Vn
    assert_same_state(ring.to_pytree(), expect)
    # the loaded rows step as the pytree forward of the loaded state
    f = torch.randint(0, 256, (2, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.tensor([False, True])
    torch.manual_seed(7)
    ac0, st0, r0 = pol.act({"img": f}, first, new, return_pd=True)
    torch.manual_seed(7)
    ac1, _, r1 = pol.act({"img": f}, first, view, return_pd=True)
    _same_outputs(_outputs(ac0, r0, [0, 1]), _outputs(ac1, r1, [0, 1]))
    assert_same_state(view.to_pytree(), st0)
    # a ring with per-row offsets copied into another: the offsets come along; a pytree loaded over it zeroes them
    other = RingState.zeros(pol, E).load_(ring)
    assert torch.equal(other.row_off, ring.row_off) and other.row_off is not ring.row_off and int(other.off) == int(ring.off)
    assert_same_state(other.to_pytree(), ring.to_pytree())
    plain = RingState.zeros(pol, E)
    assert other.load_(plain).row_off.eq(0).all()
    assert_same_state(other.to_pytree(), plain.to_pytree())
    other.load_(ring)
    assert_same_state(other.load_(everything).to_pytree(), everything)
    assert other.row_off.eq(0).all() and int(other.off) == 0
    # a whole-ring step of a ring with per-row offsets is the pytree step of its state
    st = ring.to_pytree()
    f = torch.randint(0, 256, (E, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.tensor([False, False, True, False, False])
    torch.manual_seed(8)
    ac0, st0, r0 = pol.act({"img": f}, first, st, return_pd=True)
    torch.manual_seed(8)
    ac1, _, r1 = pol.act({"img": f}, first, ring, return_pd=True)
    _same_outputs(_outputs(ac0, r0, list(range(E))), _outputs(ac1, r1, list(range(E))))
    assert_same_state(ring.to_pytree(), st0)
    with pytest.raises(ValueError, match="inert"):
        ring.rows([0, -1]).to_pytree()
    with pytest.raises(ValueError, match="inert"):
        ring.rows([-1]).load_(pol.initial_state(1))
    with pytest.raises(ValueError, match="K / V"):
        ring.rows([0, 1]).load_(pol.initial_state(3))


def _refused(monkeypatch, exc, fn, match=None):
    rec = OpRecorder(monkeypatch)
    with pytest.raises(exc, match=match):
        fn()
    assert rec.calls == [], rec.names()


def test_calls_a_view_cannot_serve_raise_before_any_op(rows_emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(13)
    ring = RingState.zeros(pol, E)
    f3 = torch.randint(0, 256, (3, 32, 32, 3), dtype=torch.uint8, generator=g)
    first3 = torch.zeros(3, dtype=torch.bool)
    _refused(monkeypatch, ValueError, lambda: pol.act({"img": f3}, first3, ring.rows([0, 2, 0])), "twice")
    _refused(monkeypatch, ValueError, lambda: pol.act({"img": f3}, first3, ring.rows([0, 2, E])), "outside")
    _refused(monkeypatch, ValueError, lambda: pol.act({"img": f3}, first3, ring.rows([0, -2, 1])), "outside")
    for bad in ([], [[0, 1]], [0.0, 1.0], torch.tensor([True, False])):
        with pytest.raises(ValueError, match="integer"):
            ring.rows(bad)
    _refused(monkeypatch, ValueError, lambda: pol.act({"img": f3}, first3, ring.rows([0, 2])), "view of 2")
    chunk = torch.randint(0, 256, (2, 2, 32, 32, 3), dtype=torch.uint8, generator=g)
    _refused(monkeypatch, ValueError, lambda: pol({"img": chunk}, torch.zeros(2, 2, dtype=torch.bool), ring.rows([1, 3])), "t = 1")
    pol.set_autograd(True)
    _refused(monkeypatch, ValueError, lambda: pol({"img": f3[:, None]}, first3[:, None], ring.rows([0, 1, 2])), "inference")
    _refused(monkeypatch, ValueError, lambda: pol.net({"img": f3[:, None]}, ring.rows([0, 1, 2]), {"first": first3[:, None]}), "inference")
    pol.set_autograd(False)
    with pytest.raises(ValueError, match="inference"):
        BCTrainer(pol).loss_and_grad(f3[:, None], first3[:, None], ring.rows([0, 1, 2]),
                                     {"camera": torch.zeros(3, 1, 1, dtype=torch.long), "buttons": torch.zeros(3, 1, 1, dtype=torch.long)})
    pol.set_precision("fp32")
    _refused(monkeypatch, NotImplementedError, lambda: pol.act({"img": f3}, first3, ring.rows([0, 1, 2])))
    pol.set_precision("bf16")
    assert ring.row_off is None and int(ring.off) == 0 and all(not m.any() for m in ring.mask)
    # GraphedAct(envs=E) steps views of its own ring only (the refusal comes before any copy; built without a GPU from its parts)
    step = GraphedAct.__new__(GraphedAct)
    step.envs, step.B, step.memory = E, 4, "ring"
    step.state = RingState.zeros(pol, E)
    _refused(monkeypatch, ValueError, lambda: step({"img": f3}, first3, ring.rows([0, 1, 2])), "own ring")
    _refused(monkeypatch, ValueError, lambda: step({"img": f3}, first3, step.state), "own ring")
    tree = step.state.to_pytree()
    _refused(monkeypatch, ValueError, lambda: step({"img": f3}, first3, tree), "own ring")
    f5 = torch.zeros(5, 32, 32, 3, dtype=torch.uint8)
    _refused(monkeypatch, ValueError, lambda: step({"img": f5}, torch.zeros(5, dtype=torch.bool), step.state.rows([0, 1, 2, 3, 4])), "batch size")
    _refused(monkeypatch, ValueError, lambda: step({"img": f3}, first3, step.state.rows([0, 1])), "3 frames")
    with pytest.raises(ValueError, match="envs"):
        GraphedAct(pol, 2, memory="pytree", envs=E)
    assert isinstance(ring.rows([1]), RingRows)
