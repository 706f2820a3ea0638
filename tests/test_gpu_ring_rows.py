"""Asynchronous rollouts through the CUDA kernels at 2x width (hidsize 2048, 16 heads, 128x128 frames): steps of any subset of a
`RingState`'s environments, through `ring.rows(idx)`, eagerly and with `GraphedAct(envs=E)`, against the pytree forward of those
environments' states gathered into a batch, bit for bit: sampled actions under a fixed seed, log-probs, vpred, every pd row and the
materialised states.  maxlen 128 (attention.cuh), 200 (64-key tiles wrap mid-tile) and 1920 (attention_long.cuh, the t = 1 band split
across a thread-block cluster), E = 3 and 64.  Each run starts from random bf16-exact full memories with random masks, with `off` and
every environment's `row_off` a few steps before their wrap; whole-ring steps, singletons, all E in permuted order and subsets padded
with -1 take turns, with episode resets.  The eager view steps run with every buffer they allocate filled with 0xFF (NaN) and again
without; environments a step does not list must keep every byte.  A graphed call of k < B rows must equal the eager call on the same
view padded with -1 rows and zero frames, and both the pytree forward of the gathered states padded the same way (inert rows: the
initial state): the GEMMs pick their kernel by the number of rows, so a padded step is compared with a padded reference."""
import pytest
import torch

from test_gpu_ring_state import _nan_buffers, _policy, _start, _step
from test_ring_rows import EnvStates, _outputs, _same_outputs
from video_pre_training_b200 import _native as nat
from video_pre_training_b200.policy import GraphedAct, RingState

pytestmark = pytest.mark.gpu


def _ring_at(pol, start, off, row_off):
    """A ring holding `start` with `off` and per-environment offsets `row_off` (memory row j of e at (off + row_off[e] + j) % maxlen)."""
    ring = RingState.from_pytree(pol, start)
    maxlen = ring.k[0].shape[1]
    for e, ro in enumerate(row_off):
        shift = (off + ro) % maxlen
        for buf in ring.k + ring.v + ring.mask:
            buf[e] = torch.roll(buf[e], shift, dims=0)
    ring.off.fill_(off)
    ring._alloc_row_off().copy_(torch.tensor(row_off, dtype=torch.int32))
    return ring


def _schedule(E, Bg, g):
    """The environments each step lists, in call order (None: the whole ring; -1: an inert padding row)."""
    perm = torch.randperm(E, generator=g).tolist()
    if E == 3:
        return [None, [2], perm, [0, -1], None, [2, 0], [1], [-1, 1, 2]]
    return [None, [37], perm, perm[:Bg], [5, -1, 63, 0, -1], None, perm[Bg:2 * Bg], [63]]


def _live(envs):
    return [i for i, e in enumerate(envs) if e >= 0]


def _same_rows(ring_a, ring_b, envs):
    real = [e for e in envs if e >= 0]
    for (m0, (k0, v0)), (m1, (k1, v1)) in zip(ring_a.rows(real).to_pytree(), ring_b.rows(real).to_pytree()):
        assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(v0, v1)


def _same_ref(ring, ref, envs):
    real = [e for e in envs if e >= 0]
    for (m0, (k0, v0)), (m1, (k1, v1)) in zip(ref.gather(real), ring.rows(real).to_pytree()):
        assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(v0, v1)


@pytest.mark.parametrize("E", [3, 64])
@pytest.mark.parametrize("maxlen", [128, 200, 1920])
def test_async_rollout_is_bit_identical_to_the_gathered_pytree_forward(maxlen, E):
    pol = _policy(maxlen)
    assert pol.net.cfg.maxlen == maxlen and pol.net.cfg.hidsize == 2048
    g = torch.Generator().manual_seed(7 * maxlen + E)
    start = _start(pol, E, g)
    ref, ref_pad = EnvStates(start), EnvStates(start)  # the reference of the unpadded eager steps, and of the padded / graphed ones
    off0 = maxlen - 1  # `off` wraps at the first whole-ring step, each row_off within its first three steps
    row_off0 = [maxlen - 1 - (e % 3) for e in range(E)]
    ring_nan, ring_rerun, ring_pad = (_ring_at(pol, start, off0, row_off0) for _ in range(3))
    Bg = min(E, 16)
    ga = GraphedAct(pol, Bg, memory="ring", envs=E)
    assert ga.state.row_off is not None
    ga.state.load_(ring_pad)
    assert torch.equal(ga.state.row_off, ring_pad.row_off)
    H = pol.net.cfg.img_shape[0]
    for s, idx in enumerate(_schedule(E, Bg, g)):
        envs = list(range(E)) if idx is None else idx
        B, live, seed = len(envs), _live(envs), 2000 + s
        frames = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, generator=g)
        first = torch.rand(B, generator=g) < 0.25
        for i, e in enumerate(envs):
            if e < 0:
                frames[i], first[i] = 0, False
        frames, first = frames.cuda(), first.cuda()
        # the reference: the pytree forward on the gathered states (inert rows: the initial state)
        ac, res, st = _step(pol.act, frames, first, ref.gather(envs), seed)
        ref.scatter(envs, st)
        want = _outputs(ac, res, live)
        del st
        # eager steps of the view (of the whole ring for None), with NaN-filled scratch buffers and again without
        untouched = torch.tensor([e for e in range(E) if e not in envs], dtype=torch.long, device="cuda")
        bufs = lambda: ring_nan.k + ring_nan.v + ring_nan.mask + [ring_nan.row_off]  # noqa: E731
        before = [x.index_select(0, untouched) for x in bufs()]
        for ring, nan in ((ring_nan, True), (ring_rerun, False)):
            rows_idx = envs if s % 2 else torch.tensor(envs, device="cuda")  # host or device idx
            state = ring if idx is None else ring.rows(rows_idx)
            ac, res, out = _step(pol.act, frames, first, state, seed, nan)
            assert out is state
            _same_outputs(want, _outputs(ac, res, live))
            assert torch.isfinite(res["log_prob"]).all()
            _same_ref(ring, ref, envs)
        assert all(torch.equal(b.view(torch.uint8), x.index_select(0, untouched).view(torch.uint8)) for b, x in zip(before, bufs()))
        del before
        # the graphed ring, against the eager call of the same view padded to the graph's batch
        if idx is not None and len(idx) <= Bg:
            k = len(idx)
            pad = list(idx) + [-1] * (Bg - k)
            f_pad = torch.zeros((Bg, H, H, 3), dtype=torch.uint8, device="cuda")
            f_pad[:k] = frames
            first_pad = torch.zeros(Bg, dtype=torch.bool, device="cuda")
            first_pad[:k] = first
            ac, res, st = _step(pol.act, f_pad, first_pad, ref_pad.gather(pad), seed)
            ref_pad.scatter(pad, st)
            want_pad = _outputs(ac, res, live)
            del st
            ac_p, res_p, _ = _step(pol.act, f_pad, first_pad, ring_pad.rows(pad), seed, True)
            ac_g, res_g, out = _step(ga, frames, first, ga.state.rows(idx), seed)
            assert out.ring is ga.state and len(out) == k
            assert all(v.shape[0] == k for v in ac_g.values()) and res_g["log_prob"].shape[0] == k
            _same_outputs(_outputs(ac_p, res_p, list(range(k))), _outputs(ac_g, res_g, list(range(k))))
            _same_outputs(want_pad, _outputs(ac_g, res_g, live))
        else:  # more rows than the graph takes: both rings step eagerly, as the unpadded reference
            ac, res, st = _step(pol.act, frames, first, ref_pad.gather(envs), seed)
            ref_pad.scatter(envs, st)
            del st
            for ring in (ring_pad, ga.state):
                ac_r, res_r, _ = _step(pol.act, frames, first, ring if idx is None else ring.rows(envs), seed)
                _same_outputs(_outputs(ac, res, live), _outputs(ac_r, res_r, live))
        _same_rows(ring_pad, ga.state, envs)
        _same_ref(ga.state, ref_pad, envs)
    for ring in (ring_nan, ring_rerun):
        _same_ref(ring, ref, list(range(E)))
    _same_ref(ga.state, ref_pad, list(range(E)))
    _same_rows(ring_pad, ga.state, list(range(E)))
    assert int(ring_nan.off) == (off0 + 2) % maxlen
    nat.device_check()
    del ga, ring_nan, ring_rerun, ring_pad, ref, ref_pad, start
    torch.cuda.empty_cache()


def test_graphed_views_refuse_other_states():
    pol = _policy(128)
    ga = GraphedAct(pol, 4, memory="ring", envs=6)
    f = torch.zeros((2, 128, 128, 3), dtype=torch.uint8, device="cuda")
    first = torch.zeros(2, dtype=torch.bool, device="cuda")
    for bad in (RingState.zeros(pol, 6).rows([0, 1]), ga.state, ga.state.rows([0, 1]).to_pytree()):
        with pytest.raises(ValueError, match="own ring"):
            ga({"img": f}, first, bad)
    with pytest.raises(ValueError, match="batch size"):
        ga({"img": f[:1].expand(5, -1, -1, -1)}, first[:1].expand(5), ga.state.rows([0, 1, 2, 3, 4]))
    assert ga.state.row_off.eq(0).all() and all(not m.any() for m in ga.state.mask)
    with _nan_buffers():
        ac, out, res = ga({"img": f}, first, ga.state.rows([5, 2]))
    assert out.envs == [5, 2] and torch.isfinite(res["log_prob"]).all()
    assert ga.state.row_off.tolist() == [0, 0, 1, 0, 0, 1] and int(ga.state.off) == 0
    del ga
    torch.cuda.empty_cache()
