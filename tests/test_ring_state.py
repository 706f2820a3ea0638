"""`RingState`, the recurrent state that a t = 1 forward updates in place, on the CPU through the test-only torch emulation of the ops
(tests/emu_ring_ops.py for the ring kernels): rollouts through a ring equal the pytree rollouts step by step (actions, log-probs, vpred,
pd and `to_pytree()` against `state_out`), past `maxlen` steps so that the offset wraps and with per-env episode resets; the pytree ->
ring -> pytree round trip; and every call a ring cannot serve raises before any op.  tests/test_gpu_ring_state.py repeats the rollouts
through the CUDA kernels at 2x width."""
import pytest
import torch

import emu_ring_ops
import vpt_b200
from common import make_policy, small_kwargs
from test_autograd import emulated  # noqa: F401  (fixture)
from test_idm_training import make_idm
from test_latents import OpRecorder
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import RingState
from video_pre_training_b200.training import BCTrainer


@pytest.fixture()
def ring_emu(emulated, monkeypatch):  # noqa: F811
    for name in ("ring_write", "attention_ring", "ring_advance"):
        monkeypatch.setattr(ops, name, getattr(emu_ring_ops, name))
    yield


def random_state(g, pol, B, exact=True):
    """A full memory with a random mask; bf16-exact K / V unless exact=False."""
    cfg = pol.net.cfg
    st = []
    for _ in range(cfg.n_layers):
        kv = [torch.randn(B, cfg.maxlen, cfg.hidsize, generator=g) for _ in range(2)]
        if exact:
            kv = [x.bfloat16().float() for x in kv]
        st.append((torch.rand(B, 1, cfg.maxlen, generator=g) < 0.7, tuple(kv)))
    return st


def _mask(m, B, maxlen):
    return torch.zeros(B, 1, maxlen, dtype=torch.bool) if m is None else m.reshape(B, 1, maxlen)


def assert_same_state(a, b):
    assert len(a) == len(b)
    for (ma, (ka, va)), (mb, (kb, vb)) in zip(a, b):
        B, maxlen = ka.shape[:2]
        assert torch.equal(_mask(ma, B, maxlen), _mask(mb, B, maxlen))
        assert ka.dtype == kb.dtype == torch.float32 and torch.equal(ka, kb) and torch.equal(va, vb)


def inputs(g, B, steps, resets):
    frames = torch.randint(0, 256, (steps, B, 32, 32, 3), dtype=torch.uint8, generator=g)
    firsts = torch.zeros(steps, B, dtype=torch.bool)
    for s, b in resets:
        firsts[s, b] = True
    return frames, firsts


def rollout(fn, state, frames, firsts, seed=100):
    """Per step (actions, log_prob, vpred, pd, the state in reference format); stochastic sampling under a fixed seed per step."""
    out = []
    for s, (f, first) in enumerate(zip(frames, firsts)):
        torch.manual_seed(seed + s)
        ac, state, res = fn({"img": f}, first, state, return_pd=True)
        out.append((ac, res, state.to_pytree() if isinstance(state, RingState) else state))
    return out, state


def assert_same_rollout(a, b):
    for (ac0, r0, s0), (ac1, r1, s1) in zip(a, b):
        assert ac0.keys() == ac1.keys() and all(torch.equal(ac0[k], ac1[k]) for k in ac0)
        assert torch.equal(r0["log_prob"], r1["log_prob"]) and torch.equal(r0["vpred"], r1["vpred"])
        assert all(torch.equal(r0["pd"][k], r1["pd"][k]) for k in r0["pd"])
        assert_same_state(s0, s1)


@pytest.mark.parametrize("start", ["initial", "random"])
def test_ring_rollout_is_the_pytree_rollout(ring_emu, start):
    """20 steps at maxlen 8: the offset wraps twice; env 1 restarts at step 3, env 0 at step 11, env 2 at steps 11 and 12."""
    pol, _, _ = make_policy(small_kwargs())
    assert pol.net.cfg.maxlen == 8
    g = torch.Generator().manual_seed(1)
    B = 3
    st0 = pol.initial_state(B) if start == "initial" else random_state(g, pol, B)
    frames, firsts = inputs(g, B, 20, [(3, 1), (11, 0), (11, 2), (12, 2)])
    ref, _ = rollout(pol.act, st0, frames, firsts)
    ring = RingState.zeros(pol, B) if start == "initial" else RingState.from_pytree(pol, st0)
    got, ring_out = rollout(pol.act, ring, frames, firsts)
    assert ring_out is ring and int(ring.off) == 20 % 8
    assert_same_rollout(ref, got)


def test_ring_forward_v_and_latents(ring_emu):
    """`forward`, `get_output_for_observation` and `v` with a ring, from frames and from cached latents, each a step of the same rollout."""
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(2)
    B = 2
    st = random_state(g, pol, B)
    ring = RingState.from_pytree(pol, st)
    frames, firsts = inputs(g, B, 11, [(4, 0)])
    for s, (f, first) in enumerate(zip(frames, firsts)):
        kind = s % 3
        if kind == 0:
            ob = {"img": f[:, None]} if s % 2 else {"img_latent": pol.encode(f[:, None])}
            (pd0, v0, _), st = pol(ob, first[:, None], st)
            (pd1, v1, _), out = pol(ob, first[:, None], ring)
        elif kind == 1:
            ob = {"img": f} if s % 2 else {"img_latent": pol.encode(f[:, None])[:, 0]}
            pd0, v0, st = pol.get_output_for_observation(ob, st, first)
            pd1, v1, out = pol.get_output_for_observation(ob, ring, first)
        else:
            v0 = pol.v({"img": f}, first, st)
            st = pol(({"img": f[:, None]}), first[:, None], st)[1]  # v drops the state: take it from the same step
            v1 = pol.v({"img": f}, first, ring)
            pd0 = pd1 = {}
            out = ring
        assert out is ring
        assert torch.equal(v0, v1) and all(torch.equal(pd0[k], pd1[k]) for k in pd0)
        if kind != 2:
            assert_same_state(st, ring.to_pytree())


def test_pytree_ring_pytree_round_trip(ring_emu):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(3)
    exact = random_state(g, pol, 2)
    assert_same_state(RingState.from_pytree(pol, exact).to_pytree(), exact)
    loose = random_state(g, pol, 2, exact=False)
    rounded = [(m, (k.bfloat16().float(), v.bfloat16().float())) for m, (k, v) in loose]
    assert_same_state(RingState.from_pytree(pol, loose).to_pytree(), rounded)  # fp32 -> bf16 as the pytree forward rounds it
    bf16 = [(m, (k.bfloat16(), v.bfloat16())) for m, (k, v) in loose]
    assert_same_state(RingState.from_pytree(pol, bf16).to_pytree(), rounded)
    empty = RingState.from_pytree(pol, pol.initial_state(2))
    assert_same_state(empty.to_pytree(), pol.initial_state(2))
    assert all(not m.any() for m in empty.mask)
    # a ring copied into another keeps its offset: the same reference-format state
    ring = RingState.from_pytree(pol, exact)
    frames, firsts = inputs(g, 2, 5, [])
    for f, first in zip(frames, firsts):
        pol.act({"img": f}, first, ring)
    other = RingState.zeros(pol, 2).load_(ring)
    assert int(other.off) == 5 and other.k[0] is not ring.k[0]
    assert_same_state(other.to_pytree(), ring.to_pytree())


def _refused(monkeypatch, exc, fn, match=None):
    rec = OpRecorder(monkeypatch)
    with pytest.raises(exc, match=match):
        fn()
    assert rec.calls == [], rec.names()


def test_calls_a_ring_cannot_serve_raise_before_any_op(ring_emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(4)
    B = 2
    frames, firsts = inputs(g, B, 2, [])
    ring = RingState.zeros(pol, B)
    chunk = frames.transpose(0, 1)  # (B, 2, H, W, 3)
    _refused(monkeypatch, ValueError, lambda: pol({"img": chunk}, firsts.T, ring), "t = 1")
    _refused(monkeypatch, ValueError, lambda: pol.act({"img": frames[0, :1]}, firsts[0, :1], ring), "RingState of")
    pol.set_autograd(True)
    _refused(monkeypatch, ValueError, lambda: pol({"img": frames[0][:, None]}, firsts[0][:, None], ring), "inference")
    _refused(monkeypatch, ValueError, lambda: pol.net({"img": frames[0][:, None]}, ring, {"first": firsts[0][:, None]}), "inference")
    pol.set_autograd(False)
    with pytest.raises(ValueError, match="inference"):  # the trainers take the pytree state
        BCTrainer(pol).loss_and_grad(frames[0][:, None], firsts[0][:, None], ring,
                                     {"camera": torch.zeros(B, 1, 1, dtype=torch.long), "buttons": torch.zeros(B, 1, 1, dtype=torch.long)})
    pol.set_precision("fp32")
    _refused(monkeypatch, NotImplementedError, lambda: pol.act({"img": frames[0]}, firsts[0], ring))
    pol.set_precision("bf16")
    assert int(ring.off) == 0 and all(not m.any() for m in ring.mask)
    idm, _, _ = make_idm()
    with pytest.raises(TypeError):
        RingState.zeros(idm, B)
    img_idm = torch.randint(0, 256, (B, 1, *idm.net.cfg.img_shape[:2], 3), dtype=torch.uint8, generator=g)
    _refused(monkeypatch, TypeError, lambda: idm({"img": img_idm}, first=firsts[0][:, None], state_in=ring))
    nomem = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), small_kwargs(attention_mask_style="none", attention_memory_size=8),
                                          vpt_b200.PI_HEAD_KWARGS)
    assert nomem.net.cfg.maxlen == 0
    with pytest.raises(ValueError, match="KV memory"):
        RingState.zeros(nomem, B)
    with pytest.raises(ValueError, match="memory"):
        vpt_b200.policy.GraphedAct(pol, B, memory="flat")
