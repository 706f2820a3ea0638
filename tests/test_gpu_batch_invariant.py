"""The batch-invariant mode on the CUDA kernels (`MinecraftAgentPolicy.set_batch_invariant`): every output of a row of a one-frame step
equals, bit for bit, the default-mode B = 1 step of that environment alone, whatever the batch size, the row's position, the other rows and
the padding, eager or graphed, pytree or ring or view.  At 2x and 1x width, maxlen 128 and 1920 (the long band's cluster split), B in
{1, 2, 3, 8, 9, 64} and each model's CNN plan boundaries read from the C ABI; three probe environments with random full memories sit at
random rows among other random rows.  Also: an asynchronous schedule run twice with other ready sets and graph batch sizes gives every
environment the same trajectory, sampled actions and `RingState.steps` included; the keyed Gumbel-max against a numpy Philox4x32-10 and a
chi-square test; and the default mode's launches unchanged after the mode was on."""
import numpy as np
import pytest
import scipy.stats
import torch

import emu_invariant_ops
import vpt_b200
from common import perturb
from test_gpu_ring_state import _nan_buffers
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import GraphedAct, RingState

pytestmark = pytest.mark.gpu

_POL = {}


def _policy(width, maxlen):
    if (width, maxlen) not in _POL:
        _POL.clear()
        torch.cuda.empty_cache()
        torch.manual_seed(0)
        kw = vpt_b200.policy_kwargs(width, attention_memory_size=maxlen + 128)
        pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
        perturb(pol)
        _POL[(width, maxlen)] = pol.cuda()
    return _POL[(width, maxlen)]


def plan_boundaries(pol):
    """The frame counts around each CNN plan boundary of this model (last small-call count and the next), from the C ABI."""
    lib, cfg = nat.lib(), pol.net.cfg
    H, W = cfg.img_shape[0], cfg.img_shape[1]
    chunk = pol.net.cnn_chunk_frames
    counts = set()
    for c in cfg.chans:
        for probe in (lambda F: lib.vpt_conv_zp_stat_parts(F, H, W, c), lambda F: lib.vpt_conv_zp_stat_parts(F, H // 2, W // 2, c),
                      lambda F: lib.vpt_pool_chan_parts(F, H, W, c), lambda F: lib.vpt_pool_stat_parts(F, H, W, c)):
            at = probe(chunk)
            small = [F for F in range(1, chunk) if probe(F) != at]
            if small:
                counts |= {max(small), max(small) + 1}
        H, W = H // 2, W // 2
    return sorted(counts)


def _start(pol, E, g):
    cfg = pol.net.cfg
    return [((torch.rand(E, 1, cfg.maxlen, generator=g) < 0.8).cuda(),
             tuple(torch.randn(E, cfg.maxlen, cfg.hidsize, generator=g).cuda().bfloat16().float() for _ in range(2))) for _ in range(cfg.n_layers)]


def _rows(state, idx):
    i = torch.as_tensor(idx, device="cuda")
    return [(m[i], (k[i], v[i])) for m, (k, v) in state]


def _frames(pol, n, g):
    H = pol.net.cfg.img_shape[0]
    return torch.randint(0, 256, (n, H, H, 3), dtype=torch.uint8, generator=g).cuda()


def _taken(pol, n, g):
    return {name: torch.randint(0, n_ac, (n, 1), generator=g).cuda() for name, (_, n_ac) in pol.head_specs.items()}


def _out(res, st, rows, ring=False):
    """(pd, vpred, log_prob, state rows) of the given batch rows; ring: `st` is a ring or view whose rows are read as a pytree."""
    pd = {k: v[rows].clone() for k, v in res["pd"].items()}
    if ring:
        state = st.to_pytree() if isinstance(st, RingState) else None
    else:
        state = st
    srows = None if state is None else [(m[rows].clone(), (k[rows].clone(), v[rows].clone())) for m, (k, v) in state]
    return pd, res["vpred"][rows].clone(), res["log_prob"][rows].clone(), srows


def _same(a, b, what):
    (pd0, v0, lp0, s0), (pd1, v1, lp1, s1) = a, b
    assert all(torch.equal(pd0[k], pd1[k]) for k in pd0), what
    assert torch.equal(v0, v1) and torch.equal(lp0, lp1), what
    if s0 is not None and s1 is not None:
        for (m0, (k0, vv0)), (m1, (k1, vv1)) in zip(s0, s1):
            assert torch.equal(m0.reshape(m1.shape), m1) and torch.equal(k0, k1) and torch.equal(vv0, vv1), what


def _ring_with_offsets(pol, start, row_off):
    """A ring holding `start` with per-environment offsets: memory row j of environment e at physical row (row_off[e] + j) % maxlen."""
    ring = RingState.from_pytree(pol, start)
    maxlen = ring.k[0].shape[1]
    src = (torch.arange(maxlen, device="cuda")[None, :] - row_off[:, None].long()) % maxlen
    for buf in ring.k + ring.v:
        buf.copy_(torch.gather(buf, 1, src[:, :, None].expand_as(buf)))
    for buf in ring.mask:
        buf.copy_(torch.gather(buf, 1, src))
    ring._alloc_row_off().copy_(row_off)
    return ring


@pytest.mark.parametrize("maxlen", [128, 1920])
@pytest.mark.parametrize("width", ["2x", "1x"])
def test_rows_equal_the_one_environment_step(width, maxlen):
    pol = _policy(width, maxlen)
    g = torch.Generator().manual_seed(hash((width, maxlen)) % 1000)
    batches = sorted({1, 2, 3, 8, 9, 64} | set(plan_boundaries(pol)))
    E = max(batches) + 3
    start = _start(pol, E, g)
    frames, first, taken = _frames(pol, E, g), (torch.rand(E, generator=g) < 0.2).cuda(), _taken(pol, E, g)
    probes = torch.randperm(E, generator=g)[:3].tolist()
    # the default-mode B = 1 step of each probe environment alone
    pol.set_batch_invariant(False)
    ref = {}
    for e in probes:
        _, st, res = pol.act({"img": frames[e:e + 1]}, first[e:e + 1], _rows(start, [e]), taken_action={k: v[e:e + 1] for k, v in taken.items()},
                             return_pd=True)
        ref[e] = _out(res, st, [0])
    pol.set_batch_invariant(True, seed=3)
    row_off = torch.randint(0, maxlen, (E,), generator=g, dtype=torch.int32).cuda()
    for B in batches:
        others = [e for e in torch.randperm(E, generator=g).tolist() if e not in probes]
        np_ = min(B, 3)
        envs = others[:B - np_]
        pos = sorted(torch.randperm(B, generator=g)[:np_].tolist())
        for p, e in zip(pos, probes[:np_]):
            envs.insert(p, e)
        where = {e: envs.index(e) for e in probes[:np_]}
        tk = {k: v[envs] for k, v in taken.items()}
        for nan in (True, False):
            with _nan_buffers() if nan else torch.no_grad():
                _, st, res = pol.act({"img": frames[envs]}, first[envs], _rows(start, envs), taken_action=tk, return_pd=True)
                for e, b in where.items():
                    _same(_out(res, st, [b]), ref[e], f"pytree B={B} env {e} nan={nan}")
                ring = RingState.from_pytree(pol, _rows(start, envs))
                _, ring, res = pol.act({"img": frames[envs]}, first[envs], ring, taken_action=tk, return_pd=True)
                st = ring.to_pytree()
                for e, b in where.items():
                    _same(_out(res, st, [b]), ref[e], f"ring B={B} env {e} nan={nan}")
            # a view of the big ring, with two inert rows among the listed ones
            venvs = list(envs)
            for _ in range(2):
                venvs.insert(int(torch.randint(0, len(venvs) + 1, (1,), generator=g)), -1)
            vrows = [i for i, e in enumerate(venvs) if e >= 0]
            vf = torch.zeros((len(venvs), *frames.shape[1:]), dtype=torch.uint8, device="cuda")
            vf[vrows] = frames[envs]
            vfirst = torch.zeros(len(venvs), dtype=torch.bool, device="cuda")
            vfirst[vrows] = first[envs]
            vtk = {k: torch.zeros((len(venvs), 1), dtype=torch.int64, device="cuda") for k in taken}
            for k in vtk:
                vtk[k][vrows] = tk[k]
            big = _ring_with_offsets(pol, start, row_off)
            snap = {e: (big.rows([e]).to_pytree(), int(big.row_off[e])) for e in range(E) if e not in envs}
            with _nan_buffers() if nan else torch.no_grad():
                _, view, res = pol.act({"img": vf}, vfirst, big.rows(venvs), taken_action=vtk, return_pd=True)
            after = big.rows(probes[:np_]).to_pytree()
            for i, e in enumerate(probes[:np_]):
                b = venvs.index(e)
                pd, v, lp, _ = _out(res, None, [b], ring=True)
                _same((pd, v, lp, [(m[i:i + 1], (k[i:i + 1], vv[i:i + 1])) for m, (k, vv) in after]), ref[e], f"view B={B} env {e} nan={nan}")
            for e, (s0, ro) in list(snap.items())[:8]:  # environments the step does not list keep every byte
                assert int(big.row_off[e]) == ro
                for (m0, (k0, v0)), (m1, (k1, v1)) in zip(s0, big.rows([e]).to_pytree()):
                    assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(v0, v1)
    pol.set_batch_invariant(False)


def _rows_of(pd, v, st, b):
    return ({k: x[b].clone() for k, x in pd.items()}, v[b].clone(),
            [(m[b].reshape(-1).clone(), (k[b].clone(), vv[b].clone())) for m, (k, vv) in st])


def _same_rows(a, b, what):
    (pd0, v0, s0), (pd1, v1, s1) = a, b
    assert pd0.keys() == pd1.keys() and all(torch.equal(pd0[k], pd1[k]) for k in pd0), what
    assert torch.equal(v0, v1), what
    for (m0, (k0, vv0)), (m1, (k1, vv1)) in zip(s0, s1):
        assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(vv0, vv1), what


@pytest.mark.parametrize("maxlen", [128, 1920])
def test_other_entry_points_equal_the_one_environment_step(maxlen):
    """`get_output_for_observation` from latents and from frames, `v`, and `forward` with T = 1: each probe row equals the same entry
    point's default-mode B = 1 call on that environment alone."""
    pol = _policy("2x", maxlen)
    g = torch.Generator().manual_seed(3 * maxlen + 1)
    E = 67
    start = _start(pol, E, g)
    frames, first = _frames(pol, E, g), (torch.rand(E, generator=g) < 0.2).cuda()
    pol.set_batch_invariant(False)
    lat = pol.encode(frames[:, None])  # (encode is batch-invariant already)
    probes = torch.randperm(E, generator=g)[:3].tolist()

    def calls(idx):
        i = torch.as_tensor(idx, device="cuda")
        st = _rows(start, idx)
        pd, v, so = pol.get_output_for_observation({"img_latent": lat[i, 0]}, st, first[i])
        out = {"latents": (pd, v, so)}
        pd, v, so = pol.get_output_for_observation({"img": frames[i]}, st, first[i])
        out["frames"] = (pd, v, so)
        out["v"] = ({}, pol.v({"img": frames[i]}, first[i], st), [])
        (pd, v, _), so = pol({"img": frames[i][:, None]}, first[i][:, None], st)
        out["forward"] = (pd, v, so)
        return out

    ref = {e: {k: _rows_of(*o, 0) for k, o in calls([e]).items()} for e in probes}
    pol.set_batch_invariant(True, seed=8)
    for B in (9, 64):
        envs = [e for e in torch.randperm(E, generator=g).tolist() if e not in probes][:B - 3]
        for p, e in zip(sorted(torch.randperm(B, generator=g)[:3].tolist()), probes):
            envs.insert(p, e)
        for k, o in calls(envs).items():
            for e in probes:
                _same_rows(_rows_of(*o, envs.index(e)), ref[e][k], f"{k} B={B} env {e}")
    pol.set_batch_invariant(False)


@pytest.mark.parametrize("maxlen", [128, 1920])
def test_graphed_rows_equal_the_one_environment_step(maxlen):
    """GraphedAct(envs=E) at two graph sizes, subsets in several orders with padding: each probe row equals the eager default B = 1 step."""
    pol = _policy("2x", maxlen)
    g = torch.Generator().manual_seed(maxlen)
    E = 24
    start = _start(pol, E, g)
    frames, first = _frames(pol, E, g), (torch.rand(E, generator=g) < 0.2).cuda()
    pol.set_batch_invariant(False)
    ref = {}
    for e in range(E):
        _, st, res = pol.act({"img": frames[e:e + 1]}, first[e:e + 1], _rows(start, [e]), stochastic=False, return_pd=True)
        ref[e] = _out(res, st, [0])
    pol.set_batch_invariant(True, seed=5)
    for Bg in (9, 16):
        ga = GraphedAct(pol, Bg, memory="ring", envs=E)
        for trial in range(3):
            ga.state.load_(start)
            k = int(torch.randint(1, Bg + 1, (1,), generator=g))
            envs = torch.randperm(E, generator=g)[:k].tolist()
            ac, view, res = ga({"img": frames[envs]}, first[envs], ga.state.rows(envs), stochastic=False, return_pd=True)
            after = ga.state.rows(envs).to_pytree()
            for i, e in enumerate(envs):
                pd, v, lp, _ = _out(res, None, [i], ring=True)
                _same((pd, v, lp, [(m[i:i + 1], (kk[i:i + 1], vv[i:i + 1])) for m, (kk, vv) in after]), ref[e], f"graph B={Bg} env {e}")
    pol.set_batch_invariant(False)


def test_schedule_independence():
    """An asynchronous schedule over E environments run twice, with other ready sets per step and other graph batch sizes (and eager
    steps in the second run): every environment's trajectory (sampled actions, log-probs, values) and final ring rows and steps agree."""
    pol = _policy("2x", 128)
    pol.set_batch_invariant(True, seed=77)
    E, S = 12, 4
    g = torch.Generator().manual_seed(9)
    start = _start(pol, E, g)
    frames = [_frames(pol, S, g) for _ in range(E)]
    firsts = [(torch.rand(S, generator=g) < 0.2).cuda() for _ in range(E)]

    def run(Bg, seed, eager_every):
        rg = torch.Generator().manual_seed(seed)
        ga = GraphedAct(pol, Bg, memory="ring", envs=E)
        ga.state.load_(start)
        ga.state._alloc_steps()
        done, traj, call = [0] * E, {e: [] for e in range(E)}, 0
        while min(done) < S:
            ready = [e for e in torch.randperm(E, generator=rg).tolist() if done[e] < S][:int(torch.randint(1, Bg + 1, (1,), generator=rg))]
            img = torch.stack([frames[e][done[e]] for e in ready])
            fst = torch.stack([firsts[e][done[e]] for e in ready])
            untouched = [e for e in range(E) if e not in ready][:3]
            before = {e: ga.state.rows([e]).to_pytree() for e in untouched}
            steps_before = ga.state.steps.clone()
            if eager_every and call % eager_every == 0:
                ac, _, res = pol.act({"img": img}, fst, ga.state.rows(ready))
            else:
                ac, _, res = ga({"img": img}, fst, ga.state.rows(ready))
            for i, e in enumerate(ready):
                traj[e].append(({k: int(v[i]) for k, v in ac.items()}, float(res["log_prob"][i]), float(res["vpred"][i])))
                done[e] += 1
            for e in untouched:
                assert int(ga.state.steps[e]) == int(steps_before[e])
                for (m0, (k0, v0)), (m1, (k1, v1)) in zip(before[e], ga.state.rows([e]).to_pytree()):
                    assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(v0, v1)
            call += 1
        return traj, ga.state.to_pytree(), ga.state.steps.clone()

    t0, s0, c0 = run(4, 1, 0)
    t1, s1, c1 = run(12, 2, 3)
    assert t0 == t1
    assert torch.equal(c0, c1) and c0.tolist() == [S] * E
    for (m0, (k0, v0)), (m1, (k1, v1)) in zip(s0, s1):
        assert torch.equal(m0, m1) and torch.equal(k0, k1) and torch.equal(v0, v1)
    pol.set_batch_invariant(False)


@pytest.mark.parametrize("n", [121, 8641])
def test_keyed_gumbel_matches_numpy_philox(n):
    g = torch.Generator().manual_seed(n)
    rows = 256
    logits = (torch.randn(rows, n, generator=g) * 3).cuda()
    keys = torch.stack([torch.randint(0, 2 ** 40, (rows,), generator=g), torch.randint(0, 2 ** 40, (rows,), generator=g)], 1).cuda()
    for seed, head in ((0, 0), (2 ** 33 + 5, 1)):
        got = ops.gumbel_argmax_keyed(logits, keys, seed, head).cpu().numpy()
        sc = emu_invariant_ops.keyed_scores(logits, keys, seed, head)
        top2 = np.sort(sc, 1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > 1e-4
        assert clear.mean() > 0.9
        assert np.array_equal(got[clear], sc.argmax(1)[clear])
        picked = sc[np.arange(rows), got]
        assert (picked >= top2[:, 1] - 1e-4).all()  # elsewhere one of the near-ties


def test_keyed_gumbel_distribution_and_keys():
    g = torch.Generator().manual_seed(1)
    n, draws = 121, 120000
    lg = torch.log_softmax(torch.randn(n, generator=g) * 1.5, 0)
    logits = lg.expand(draws, n).contiguous().cuda()
    keys = torch.stack([torch.zeros(draws, dtype=torch.int64), torch.arange(draws)], 1).cuda()
    idx = ops.gumbel_argmax_keyed(logits, keys, 123, 1).cpu()
    counts = torch.bincount(idx, minlength=n).double().numpy()
    expect = lg.exp().double().numpy() * draws
    ok = expect >= 5
    obs_, exp_ = np.append(counts[ok], counts[~ok].sum()), np.append(expect[ok], expect[~ok].sum())
    chi2 = float(((obs_ - exp_) ** 2 / exp_).sum())
    assert scipy.stats.chi2.sf(chi2, len(obs_) - 1) > 1e-4, chi2
    # the same (seed, stream, step) gives the same action in any row; another seed or step other noise
    same = torch.tensor([[5, 9]] * 64).cuda()
    lg2 = torch.randn(n, generator=g).expand(64, n).contiguous().cuda()
    a = ops.gumbel_argmax_keyed(lg2, same, 7, 0)
    assert (a == a[0]).all()
    steps = torch.stack([torch.full((64,), 5), torch.arange(64)], 1).cuda()
    assert len(set(ops.gumbel_argmax_keyed(lg2, steps, 7, 0).tolist())) > 10
    seeds = [int(ops.gumbel_argmax_keyed(lg2[:1], same[:1], s, 0)) for s in range(64)]
    assert len(set(seeds)) > 10


INVARIANT_OPS = ("gemm_rowwise", "conv3x3_zp_plan", "maxpool3s2_plan", "attention_plan", "attention_ring_plan", "gumbel_argmax_keyed",
                 "ring_noise_keys")


def test_default_mode_unchanged(monkeypatch):
    """With the flag off, or toggled on and off, a step launches only the default kernels (none of the row-wise, `_plan` or keyed
    symbols' wrappers runs) and gives the same bits; with the flag on, it runs them."""
    called = []
    for name in INVARIANT_OPS:
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _fn=fn, _name=name, **k: (called.append(_name), _fn(*a, **k))[1])
    pol = _policy("2x", 128)
    g = torch.Generator().manual_seed(4)
    B = 9
    start = _start(pol, B, g)
    f, first = _frames(pol, B, g), (torch.rand(B, generator=g) < 0.2).cuda()
    pol.set_batch_invariant(False)

    def step():
        n0 = ops.LAUNCHES
        _, st, res = pol.act({"img": f}, first, start, stochastic=False, return_pd=True)
        return ops.LAUNCHES - n0, _out(res, st, list(range(B)))

    n_def, out_def = step()
    assert called == []
    pol.set_batch_invariant(True)
    step()
    assert {"gemm_rowwise", "conv3x3_zp_plan", "maxpool3s2_plan", "attention_plan"} <= set(called)
    called.clear()
    pol.set_batch_invariant(False)
    n_after, out_after = step()
    assert called == [] and n_after == n_def
    _same(out_after, out_def, "default after the mode")


def test_keyed_gumbel_extreme_word():
    """Seed 0, head 1, stream 0, step 881 draws the Philox word 0xffffffdc for column 8114: its uniform stays below 1, so the column
    with logit -1e4 does not win over the one with logit 50."""
    lg = torch.full((2, 8641), -10.0)
    lg[:, 8114], lg[:, 3] = -1e4, 50.0
    keys = torch.tensor([[0, 881], [0, 881]]).cuda()
    assert ops.gumbel_argmax_keyed(lg.cuda(), keys, 0, 1).tolist() == [3, 3]
