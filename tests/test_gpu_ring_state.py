"""`RingState` through the CUDA kernels at 2x width (hidsize 2048, 16 heads, 128x128 frames): eager `act` with the pytree state, eager `act`
with a RingState and `GraphedAct(memory="ring")`, step by step and bit for bit: sampled actions under a fixed seed, log-probs, vpred, every
pd row and the materialised state.  maxlen 128 (the released models: attention.cuh), 200 (the band's 64-key tiles wrap mid-tile in the
ring) and 1920 (attention_long.cuh; the t = 1 band is split across a thread-block cluster), B = 1, 3 and 64.  Each run starts from a
random bf16-exact full memory with a random mask, with the ring's offset two steps before its wrap, resets some environments on the way,
runs the ring's forward with every buffer it allocates filled with 0xFF (NaN) and runs it twice."""
import contextlib

import pytest
import torch

import vpt_b200
from common import perturb
from video_pre_training_b200 import _native as nat
from video_pre_training_b200.policy import GraphedAct, RingState

pytestmark = pytest.mark.gpu

STEPS = 4
_POL = {}


def _policy(maxlen):
    if maxlen not in _POL:
        _POL.clear()
        torch.cuda.empty_cache()
        torch.manual_seed(0)
        kw = vpt_b200.policy_kwargs("2x", attention_memory_size=maxlen + 128)
        pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
        perturb(pol)
        _POL[maxlen] = pol.cuda()
    return _POL[maxlen]


def _start(pol, B, g):
    cfg = pol.net.cfg
    st = []
    for _ in range(cfg.n_layers):
        m = (torch.rand(B, 1, cfg.maxlen, generator=g) < 0.8).cuda()
        kv = tuple(torch.randn(B, cfg.maxlen, cfg.hidsize, generator=g).cuda().bfloat16().float() for _ in range(2))
        st.append((m, kv))
    return st


def _rotated(ring, off):
    """The same reference-format state with the ring's offset at `off` (memory row j at physical row (off + j) % maxlen)."""
    for buf in ring.k + ring.v + ring.mask:
        buf.copy_(torch.roll(buf, off, dims=1))
    ring.off.fill_(off)
    return ring


@contextlib.contextmanager
def _nan_buffers():
    """torch.empty / empty_like return 0xFF-filled memory (NaN in bf16 and fp32) while active."""
    empty, empty_like = torch.empty, torch.empty_like

    def fill(t):
        if t.numel():
            t.view(-1).view(torch.uint8).fill_(0xFF) if t.is_contiguous() else t.fill_(float("nan"))
        return t

    torch.empty = lambda *a, **k: fill(empty(*a, **k))
    torch.empty_like = lambda *a, **k: fill(empty_like(*a, **k))
    try:
        yield
    finally:
        torch.empty, torch.empty_like = empty, empty_like


def _step(fn, f, first, state, seed, nan=False):
    torch.manual_seed(seed)
    with _nan_buffers() if nan else contextlib.nullcontext():
        ac, st, res = fn({"img": f}, first, state, return_pd=True)
    return {k: v.clone() for k, v in ac.items()}, {k: (v.clone() if torch.is_tensor(v) else {n: x.clone() for n, x in v.items()}) for k, v in res.items()}, st


def _same_out(a, b):
    (ac0, r0), (ac1, r1) = a, b
    assert ac0.keys() == ac1.keys() and all(torch.equal(ac0[k], ac1[k]) for k in ac0)
    assert torch.equal(r0["log_prob"], r1["log_prob"]) and torch.equal(r0["vpred"], r1["vpred"])
    assert r0["pd"].keys() == r1["pd"].keys() and all(torch.equal(r0["pd"][k], r1["pd"][k]) for k in r0["pd"])
    assert torch.isfinite(r0["log_prob"]).all()


def _same_state(ref, ring):
    got = ring.to_pytree()
    for (m0, (k0, v0)), (m1, (k1, v1)) in zip(ref, got):
        assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(v0, v1)
    del got


RESETS = {1: [(1, 0)], 3: [(0, 1), (2, 2), (3, 1)], 64: [(1, b) for b in range(0, 64, 5)] + [(3, 7)]}


@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("maxlen", [128, 200, 1920])
def test_ring_rollout_is_bit_identical_to_the_pytree_rollout(maxlen, B):
    pol = _policy(maxlen)
    assert pol.net.cfg.maxlen == maxlen and pol.net.cfg.hidsize == 2048
    g = torch.Generator().manual_seed(maxlen + B)
    start = _start(pol, B, g)
    frames = torch.randint(0, 256, (STEPS, B, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    firsts = torch.zeros(STEPS, B, dtype=torch.bool)
    for s, b in RESETS[B]:
        firsts[s, b] = True
    firsts = firsts.cuda()
    off0 = maxlen - 2  # the offset wraps after the second step
    ring_nan = _rotated(RingState.from_pytree(pol, start), off0)
    ring_rerun = _rotated(RingState.from_pytree(pol, start), off0)
    ga = GraphedAct(pol, B, memory="ring")
    ga_state = _rotated(RingState.from_pytree(pol, start), off0)  # copied into the graph's ring on the first call
    st = start
    step0 = None
    for s in range(STEPS):
        f, first, seed = frames[s], firsts[s], 1000 + s
        *ref, st = _step(pol.act, f, first, st, seed)
        step0 = step0 or ref
        for fn, ring, nan in ((pol.act, ring_nan, True), (pol.act, ring_rerun, False), (ga, ga_state, True)):
            *out, ring_out = _step(fn, f, first, ring, seed, nan)
            _same_out(ref, out)
            _same_state(st, ring_out)
        ga_state = ga.state
        assert int(ring_nan.off) == (off0 + s + 1) % maxlen
    assert ga_state is ga.state and int(ga.state.off) == int(ring_nan.off)
    # a pytree passed to the graphed ring is copied in: the first step again
    *out, ring_out = _step(ga, frames[0], firsts[0], start, 1000)
    _same_out(step0, out)
    assert ring_out is ga.state and int(ga.state.off) == 1
    nat.device_check()
    del ga, ring_nan, ring_rerun, st, start
    torch.cuda.empty_cache()
