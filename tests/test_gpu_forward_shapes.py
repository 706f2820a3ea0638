"""Forward kernels of the inference path at the shapes the released models run (1x / 2x / 3x widths and the 4x IDM), each on isolated
inputs at its own launch plan, against the float64 unfused layers of tests/fwd_refs.py (the oracle's GroupNorm -> conv -> ReLU, LayerNorm
-> linear, attention), with the product's own fold tables (`policy._Prepared`) -- so the folds are under test with the epilogues.

Every call also keeps the buffer contract: outputs, statistics partials and fold tables are filled with 0xFF (a NaN) inside NaN guard
bands and must come back finite inside (ZP pad row / column = 0, every partial slot the finaliser reads written) and untouched outside;
inputs sit inside NaN guard bands too, so a finite output proves nothing was read outside them; two identical calls give identical bits
(large activations are compared through a position-weighted int64 digest of their bit patterns per frame).

The CNN ops run at the production chunk (2048 frames, 512 for the IDM) and at a ragged last chunk, and compare the float64 reference on
a fixed set of frames: the first, the last, and three between.  Besides randn frames, the inputs hold post-ReLU-like frames whose mean
is several times their spread and one frame whose spread is 1 / 64 of its mean (the inputs where a GroupNorm fold cancels most of its
bits); each check prints its error per kind of frame beside its bound, and the peak device memory of each test."""
import ctypes as C
import gc

import pytest
import torch
import torch.nn.functional as F

import fwd_refs as Rf
from test_gpu_backward_shapes import Guarded, _run_twice, check_bf16, check_sum
from test_gpu_long_attention import fwd_ref as attention_ref
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops, ops_ring
from video_pre_training_b200.policy import NBASIS, _dense_from_zp

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
SHAPES = {w: Rf.forward_shapes(w) for w in Rf.MODELS}

# Bounds: each is at most 4x the worst value measured on an H100 80GB HBM3 (SXM, 700 W power limit), given beside it.  bf16 outputs: |err| <= 2^-8 |ref| +
# floor * (max |ref| of the pixel / row); the floor covers the bf16 rounding of the folded weights (W * gamma), which the float64 layer
# does not have.
CONV_FLOOR = 1e-2      # every conv / pool / norm output, randn, DC-shifted and near-constant frames alike; measured 4.8e-3
LIN_FLOOR = 8e-3       # linear folds and the Q / K / V segments; measured 3.2e-3
# The dense layer (K = (Hf+1)(Wf+1)C2 = 37k .. 148k) on the tensor-core kernel, for a row whose spread is 1/64 of its mean: the
# LayerNorm fold cancels rstd * (x . W) against rstd * mean * S1, and the fp32 accumulation error of x . W grows with K; measured
# 3.1e-3 / 6.6e-3 / 1.7e-2 / 1.5e-2 (1x / 2x / 3x / IDM), rel-L2 up to 1.8e-2 (INTEGRATION.md, "Precision of the LayerNorm fold").
# Randn and DC-shifted rows (mean 6x the spread) stay within LIN_FLOOR, and so does the small-M kernel of rollout on every row.
DENSE_FLAT_FLOOR = 4e-2
ATTN_FLOOR = 5e-3      # measured 2.0e-3
STAT_MEAN, STAT_RSTD = 6e-7, 2e-6  # |d mean| * rstd and |d rstd| / rstd of a kernel's (mean, rstd) vs float64 of its stored output; measured 2.1e-7, 7.6e-7
CHAN_ELEM, CHAN_L2 = 8e-7, 2e-7    # per-channel (sum, sumsq) partials; measured 2.7e-7, 6.4e-8
HEAD_ELEM, HEAD_L2 = 1e-3, 5e-3    # fp32 logits and R: |err| / sum |terms|, rel-L2 (bf16-rounded weights); measured 3.7e-4, 1.8e-3
LOGSM_ABS = 4e-6                   # log_softmax of the stored logits, max |err|; measured 1.2e-6
FOLD_REL = 5e-5                    # norm2_fold's rstd0 * rstd1 and per-channel affine, max relative error; measured 1.6e-5


def lib():
    return nat.lib()


def stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------------------------
# models, inputs, checks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=Rf.MODELS)
def model(request):
    """(width, shapes, policy on the device, float64 net state dict on the device, the net's _Prepared); one model at a time"""
    w = request.param
    pol, sd = Rf.make_model(w)
    pol = pol.to(DEV)
    m = [w, SHAPES[w], pol, Rf.SD64(sd, DEV), pol.net.prepared()]
    yield m
    # a policy holds its weight-layout caches through bound methods of itself (`_Versioned`): a reference cycle, which only the cyclic
    # collector frees.  pytest still holds the yielded value here, so it is emptied before collecting; otherwise the model would stay on
    # the device for the tests that run after this module
    m.clear()
    del pol, sd
    _WEIGHTS.clear()
    gc.collect()
    torch.cuda.empty_cache()
    print(f"{w} model released: {torch.cuda.memory_allocated() / 2 ** 30:.2f} GiB still allocated")


@pytest.fixture(autouse=True)
def peak_memory(request):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"{request.node.name}: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


def chunks(s):
    """the production chunk, a ragged last chunk (N = chunk + 200 frames; the IDM cuts whole 128-frame sequences: 512 + 256) and the
    small calls (`small_counts`)"""
    return ((s["chunk"], 256) if s["conv3d"] else (s["chunk"], 200)) + tuple(small_counts(s))


def pool_parts(Fn, H, W, Cc):
    """statistics partials per frame of vpt_maxpool3s2 on a [Fn, H, W, Cc] input, with the per-channel partials where ops.maxpool3s2 asks
    for them"""
    return lib().vpt_pool_chan_parts(Fn, H, W, Cc) if with_chan(Cc) else lib().vpt_pool_stat_parts(Fn, H, W, Cc)


def plan_probes(s):
    """{op: Fn -> statistics partials per frame} of the CNN ops whose launch plan follows the frame count: the blocks' convolutions
    (64-column weight tiles for a few frames) and the pools of stacks 1 and 2 (more blocks per frame)"""
    probes = {}
    for i, sh in enumerate(s["stacks"]):
        H, W, Cc = sh["H"], sh["W"], sh["C"]
        probes[f"stack {i} block conv"] = lambda Fn, H=H, W=W, Cc=Cc: conv_parts(Fn, H // 2, W // 2, Cc)
        if not sh["fused_first"]:
            probes[f"stack {i} maxpool3s2"] = lambda Fn, H=H, W=W, Cc=Cc: pool_parts(Fn, H, W, Cc)
    return probes


def last_small(probe, chunk):
    """the largest frame count whose partial count differs from the production chunk's (None: every count takes the chunk's plan)"""
    at_chunk = probe(chunk)
    return max((Fn for Fn in range(1, chunk) if probe(Fn) != at_chunk), default=None)


def small_counts(s):
    """1, 3, 8 and 9 frames, and for each op of `plan_probes` the last count of its small-call plan and the first of the batch plan
    (derived from the C ABI, so the cases follow the kernels when the thresholds move)"""
    counts = {1, 3, 8, 9}
    for probe in plan_probes(s).values():
        last = last_small(probe, s["chunk"])
        if last is not None:
            counts |= {last, last + 1}
    return sorted(counts)


def check_plan(s, op, Fn):
    """prints the plan a call of Fn frames takes (its partials per frame beside the production chunk's) and asserts it at the op's own
    boundary: the small-call plan at the last count that takes it, the batch plan one frame later"""
    probe = plan_probes(s)[op]
    P, P0, last = probe(Fn), probe(s["chunk"]), last_small(probe, s["chunk"])
    print(f"{op} F={Fn}: {'small-call' if P != P0 else 'batch'} plan, {P} partials per frame ({P0} at the production chunk)")
    assert Fn != last or P != P0, (op, Fn)
    assert last is None or Fn != last + 1 or P == P0, (op, Fn)


def frame_kind(f, Fn):
    if Fn < 5:  # every kind that fits: the last frame near-constant from 3 frames on, a single frame DC-shifted (as edge_rows' single row)
        return "const" if (f == Fn - 1 and Fn >= 3) else "dc" if (f % 2 == 1 or Fn == 1) else "randn"
    return "const" if f == Fn - 1 else "dc" if (f % 2 == 1 or f == Fn - 2) else "randn"


def sel_frames(Fn):
    return sorted({f for f in (0, 1, Fn // 2, Fn - 2, Fn - 1) if 0 <= f < Fn})


def fill(t, seed, relu=False):
    """ZP bf16 frames t [F, H+1, W+1, C] (a view into a Guarded buffer): randn (|randn| with relu), odd frames and F-2 relu(randn) + 3
    (mean / spread ~ 6), the last frame 3 + randn * 3/64; zero pad row / column.  Generated in frame chunks."""
    Fn, Hp, Wp, Cc = t.shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    step = max(1, (1 << 26) // (Hp * Wp * Cc))
    for f0 in range(0, Fn, step):
        f1 = min(Fn, f0 + step)
        x = torch.randn((f1 - f0, Hp - 1, Wp - 1, Cc), generator=g, device=DEV)
        if relu:
            x = x.abs()
        for f in range(f0, f1):
            k = frame_kind(f, Fn)
            if k == "dc":
                x[f - f0] = x[f - f0].relu() + 3.0
            elif k == "const":
                x[f - f0] = 3.0 + x[f - f0] * (3.0 / 64)
        t[f0:f1, :-1, :-1] = x.to(BF16)
        t[f0:f1, -1] = 0
        t[f0:f1, :, -1] = 0
    return t


def guarded_zp(Fn, H, W, Cc, dtype=BF16):
    b = Guarded(Fn * (H + 1) * (W + 1) * Cc, dtype)
    return b, b.t.view(Fn, H + 1, W + 1, Cc)


def refill(*bufs):
    for b in bufs:
        b.raw.fill_(0xFF)


def all_finite(t):
    v = t.reshape(t.shape[0], -1)
    step = max(1, (1 << 27) // max(1, v.shape[1]))
    return all(bool(torch.isfinite(v[i:i + step]).all()) for i in range(0, v.shape[0], step))


def pads_zero(z):
    return bool((z[:, -1] == 0).all()) and bool((z[:, :, -1] == 0).all())


_WEIGHTS = {}


def digest(t):
    """per frame: sum_i bits[i] * w[i] (int64) of the 16/32-bit patterns of t[f] -- a position-weighted checksum for bit-identity checks
    of activations too large to keep two copies of"""
    v = t.reshape(t.shape[0], -1)
    v = v.view(torch.int16) if v.element_size() == 2 else v.view(torch.int32)
    n = v.shape[1]
    if _WEIGHTS.get(n) is None:
        _WEIGHTS.clear()
        _WEIGHTS[n] = torch.randint(1, 1 << 20, (n,), generator=torch.Generator(device=DEV).manual_seed(n), device=DEV, dtype=torch.int32)
    w = _WEIGHTS[n]
    step = max(1, (1 << 25) // n)
    return torch.cat([(v[i:i + step].to(torch.int64) * w).sum(1) for i in range(0, v.shape[0], step)])


def check_frames(name, out_zp, ref, idx, floor):
    """check_bf16 of the interior of the selected frames, per kind of frame (randn / dc / const)"""
    Fn = out_zp.shape[0]
    kinds = [frame_kind(f, Fn) for f in idx]
    for k in dict.fromkeys(kinds):
        j = [i for i, kk in enumerate(kinds) if kk == k]
        check_bf16(f"{name} [{k} frames]", out_zp[[idx[i] for i in j]][:, :-1, :-1], ref[j], floor)


def check_stats(name, mr, ref):
    """kernel (mean, rstd) [G][2] vs float64 (mean, rstd) of what it stored"""
    e_m = ((mr[:, 0].to(F64) - ref[:, 0]).abs() * ref[:, 1]).max().item()
    e_r = ((mr[:, 1].to(F64) - ref[:, 1]).abs() / ref[:, 1]).max().item()
    print(f"{name}: |d mean| * rstd {e_m:.2e} (bound {STAT_MEAN:.0e}), |d rstd| / rstd {e_r:.2e} (bound {STAT_RSTD:.0e})")
    assert torch.isfinite(mr).all() and e_m <= STAT_MEAN and e_r <= STAT_RSTD, name


def conv_call(x, Wb, H, W, out, part=None, mr=None, S1=None, S2=None, relu=1, residual=None, Ef=None, rs=None, rb=None):
    """vpt_conv3x3_zp into caller buffers; returns the finalised (mean, rstd) when `part` is given"""
    a = nat.ConvZpArgs()
    Fn, Cout = x.shape[0], Wb.shape[0]
    a.x, a.w, a.F, a.H, a.W, a.Cin, a.Cout = x.data_ptr(), Wb.data_ptr(), Fn, H, W, x.shape[3], Cout
    a.mr, a.S1, a.S2, a.relu, a.residual, a.out, a.stat_part = _p(mr), _p(S1), _p(S2), relu, _p(residual), out.data_ptr(), _p(part)
    a.Ef, a.res_scale, a.res_shift = _p(Ef), _p(rs), _p(rb)
    nat.check(lib().vpt_conv3x3_zp(C.byref(a), stream()), "vpt_conv3x3_zp")
    if part is None:
        return None
    return ops.stats_finalize(part, Fn, (H + 1) * (W + 1) * conv_parts(Fn, H, W, Cout), H * W * Cout)


def conv_parts(Fn, H, W, Cout):
    assert lib().vpt_conv_zp_t_stat_floats(Fn, H, W, Cout) == 0
    return lib().vpt_conv_zp_stat_parts(Fn, H, W, Cout)


def conv_part_buf(Fn, H, W, Cout):
    return Guarded(Fn * (H + 1) * (W + 1) * conv_parts(Fn, H, W, Cout) * 2)


def with_chan(Cc):
    """the pool kernels hand per-channel partials to norm2_fold (ops.maxpool3s2: C / 8 divides 256)"""
    return Cc >= 8 and 256 % (Cc // 8) == 0


def chan_sums(y_zp, parts):
    """per-channel (sum, sumsq) partials of the interior of ZP y, fp32 [F][parts][C][2]: float64 sums over `parts` runs of pixels, each
    rounded once (the shape norm2_fold reads, whatever kernel made them)"""
    yi = y_zp[:, :-1, :-1, :].to(F64).flatten(1, 2)
    return torch.stack([torch.stack([b.sum(1), (b * b).sum(1)], -1) for b in yi.tensor_split(parts, 1)], 1).float()


def in_chunks(fn, x, n=64):
    return torch.cat([fn(x[i:i + n]) for i in range(0, x.shape[0], n)])


# ---------------------------------------------------------------------------------------------------------------------
# A + B + C: the CNN
# ---------------------------------------------------------------------------------------------------------------------
def test_stack0_firstconv_pool(model):
    """u8 -> conv3x3 + bias -> ReLU -> max-pool, fused (vpt_firstconv_pool) at 128 x 128 for the model's C0: output against float64
    fanin_conv -> max_pool2d, the per-frame (mean, rstd) and the per-(tile, channel) partials against float64 sums"""
    w, s, pol, sd, prep = model
    if s["firstconv"] is None:
        pytest.skip("the IDM's stack 0 opens with the conv3d pre-stage and a normalised conv (test_stack_firstconv_and_pool)")
    st, C0 = prep.stacks[0], s["firstconv"]
    H, W = s["stacks"][0]["H"], s["stacks"][0]["W"]
    for Fn in chunks(s):
        img = torch.randint(0, 256, (Fn, H, W, 3), dtype=torch.uint8, generator=torch.Generator(device=DEV).manual_seed(Fn), device=DEV)
        img[Fn - 1] = 128 + img[Fn - 1] // 64  # a nearly flat frame
        P = lib().vpt_firstconv_stat_parts(Fn, H, W, C0)
        assert P % C0 == 0
        ob, out = guarded_zp(Fn, H // 2, W // 2, C0)
        pb = Guarded(Fn * P * 2)

        def call():
            refill(ob, pb)
            nat.check(lib().vpt_firstconv_pool(img.data_ptr(), st["fc_w"].data_ptr(), st["fc_b"].data_ptr(), out.data_ptr(), pb.ptr(), Fn, H, W, C0,
                                               1, 0, stream()), "vpt_firstconv_pool")
            return [digest(out), pb.t.clone()], [ob, pb]

        _run_twice(f"{w} firstconv_pool C0={C0} F={Fn}", call)
        assert all_finite(out) and pads_zero(out) and all_finite(pb.t)
        idx = sel_frames(Fn)
        ref = Rf.firstconv_pool(img[idx], sd, "img_process.cnn.stacks.0")
        check_frames(f"{w} firstconv_pool C0={C0} F={Fn}", out, ref, idx, CONV_FLOOR)
        mr = ops.stats_finalize(pb.t.view(Fn, P, 2), Fn, P, (H // 2) * (W // 2) * C0)
        check_stats(f"{w} firstconv_pool (mean, rstd) F={Fn}", mr[idx], Rf.stats(out[idx], zp=True))
        chan = pb.t.view(Fn, P // C0, C0, 2)[idx].sum(1)
        o = out[idx][:, :-1, :-1].to(F64)
        ref = torch.stack([o.sum((1, 2)), (o * o).sum((1, 2))], -1)
        check_sum(f"{w} firstconv_pool per-channel sums F={Fn}", chan, ref, ref.abs(), CHAN_ELEM, CHAN_L2)
        del ob, out, pb, img


def test_stack_firstconv_and_pool(model):
    """stacks 1 and 2 (and the IDM's stack 0): GroupNorm(1) -> conv3x3 -> ReLU with st["first"] (vpt_conv3x3_zp, no statistics) against
    float64 fanin_conv, then vpt_maxpool3s2 (zp, per-channel partials): bit-exact with float64 max-pool of the stored conv output"""
    w, s, pol, sd, prep = model
    for i, sh in enumerate(s["stacks"]):
        if sh["fused_first"]:
            continue
        H, W, Cin, Cc = sh["H"], sh["W"], sh["Cin"], sh["C"]
        Wb, S1, S2 = prep.stacks[i]["first"]
        p = f"img_process.cnn.stacks.{i}"
        for Fn in chunks(s):
            xb, x = guarded_zp(Fn, H, W, Cin)
            fill(x, 100 + i)
            idx = sel_frames(Fn)
            mr = in_chunks(lambda v: Rf.stats(v, zp=True), x).float()
            fb, full = guarded_zp(Fn, H, W, Cc)

            def conv():
                refill(fb)
                conv_call(x, Wb, H, W, full, mr=mr, S1=S1, S2=S2, relu=1)
                return [digest(full)], [xb, fb]

            _run_twice(f"{w} stack {i} firstconv {H}x{W} {Cin}->{Cc} F={Fn}", conv)
            assert all_finite(full) and pads_zero(full)
            check_frames(f"{w} stack {i} firstconv F={Fn}", full, Rf.conv(x[idx], sd, p + ".firstconv"), idx, CONV_FLOOR)
            del xb, x
            chan = with_chan(Cc)
            P = pool_parts(Fn, H, W, Cc)
            check_plan(s, f"stack {i} maxpool3s2", Fn)
            yb, y = guarded_zp(Fn, H // 2, W // 2, Cc)
            pb, cb = Guarded(Fn * P * 2), Guarded(Fn * P * Cc * 2 if chan else 4)

            def pool():
                refill(yb, pb, cb)
                nat.check(lib().vpt_maxpool3s2(full.data_ptr(), y.data_ptr(), pb.ptr(), cb.ptr() if chan else None, Fn, H, W, Cc, 1, stream()),
                          "vpt_maxpool3s2")
                return [digest(y), pb.t.clone(), cb.t.clone()], [fb, yb, pb, cb]

            _run_twice(f"{w} stack {i} maxpool3s2 {H}x{W}x{Cc} F={Fn}", pool)
            assert all_finite(y) and pads_zero(y) and all_finite(pb.t) and (not chan or all_finite(cb.t))
            ref = Rf.maxpool(full[idx]).to(BF16)
            bad = (y[idx][:, :-1, :-1] != ref).sum().item()
            print(f"{w} stack {i} maxpool3s2 F={Fn}: mismatches {bad} (bound 0)")
            assert bad == 0
            mr = ops.stats_finalize(pb.t.view(Fn, P, 2), Fn, P, (H // 2) * (W // 2) * Cc)
            check_stats(f"{w} stack {i} maxpool3s2 (mean, rstd) F={Fn}", mr[idx], Rf.stats(y[idx], zp=True))
            o = y[idx][:, :-1, :-1].to(F64)
            ref = torch.stack([o.sum((1, 2)), (o * o).sum((1, 2))], -1)
            if chan:
                check_sum(f"{w} stack {i} maxpool3s2 per-channel sums F={Fn}", cb.t.view(Fn, P, Cc, 2)[idx].sum(1), ref, ref.abs(), CHAN_ELEM, CHAN_L2)
            del fb, full, yb, y, pb, cb


def test_block0_with_the_stack_norm_folded(model):
    """inference block 0 (policy.py, `_cnn_chunk`): vpt_norm2_fold with st["conv0n"], conv0 with the per-frame table Ef, conv1 with the
    affine residual y1 -> against float64 GroupNorm_n -> cnn_basic_block; the (mean, rstd) of conv0 against float64 of its output"""
    w, s, pol, sd, prep = model
    for i, sh in enumerate(s["stacks"]):
        H, W, Cc = sh["H"] // 2, sh["W"] // 2, sh["C"]
        if not with_chan(Cc):
            continue  # no per-channel partials from the pool (C = 384): inference runs affine_norm_zp and block 0 unfolded
        st = prep.stacks[i]
        p = f"img_process.cnn.stacks.{i}"
        Wb0, tabs = st["conv0n"]
        Wb1, S1, S2 = st["convs"][1]
        for Fn in chunks(s):
            yb, y1 = guarded_zp(Fn, H, W, Cc)
            fill(y1, 200 + i, relu=True)
            # as many partials as the producer hands norm2_fold at this frame count: one per 8 x 8 tile from the fused first conv, the
            # pool's blocks per frame otherwise (more of them for a few frames)
            NP = lib().vpt_firstconv_stat_parts(Fn, sh["H"], sh["W"], Cc) // Cc if sh["fused_first"] else pool_parts(Fn, sh["H"], sh["W"], Cc)
            if not sh["fused_first"]:
                check_plan(s, f"stack {i} maxpool3s2", Fn)
            print(f"{w} stack {i} norm2_fold F={Fn}: {NP} per-channel partials per frame")
            chan = in_chunks(lambda v: chan_sums(v, NP), y1)
            bufs = [Guarded(Fn * 2), Guarded(Fn * 9 * Cc), Guarded(Fn * Cc), Guarded(Fn * Cc)]
            mrE, Ef, rs, rb = bufs[0].t.view(Fn, 2), bufs[1].t.view(Fn, 9, Cc), bufs[2].t.view(Fn, Cc), bufs[3].t.view(Fn, Cc)

            def fold():
                refill(*bufs)
                nat.check(lib().vpt_norm2_fold(chan.data_ptr(), NP, Cc, H * W, st["n_g"].data_ptr(), st["n_b"].data_ptr(), *[t.data_ptr() for t in tabs],
                                               Cc, 1e-5, mrE.data_ptr(), Ef.data_ptr(), rs.data_ptr(), rb.data_ptr(), Fn, stream()), "vpt_norm2_fold")
                return [b.t.clone() for b in bufs], bufs

            _run_twice(f"{w} stack {i} norm2_fold F={Fn}", fold)
            assert all(all_finite(b.t[None]) for b in bufs)
            idx = sel_frames(Fn)
            st1 = Rf.stats(y1[idx], zp=True)
            x0 = F.group_norm(Rf.nchw(y1[idx]), 1, sd[p + ".n.weight"], sd[p + ".n.bias"], eps=1e-5)
            rstd0 = Rf.stats(x0)[:, 1]
            e = max(((mrE[idx, 1].to(F64) - st1[:, 1] * rstd0) / (st1[:, 1] * rstd0)).abs().max().item(),
                    ((rs[idx].to(F64) - st1[:, 1:2] * sd[p + ".n.weight"]).abs() / (st1[:, 1:2] * sd[p + ".n.weight"]).abs()).max().item())
            shift = sd[p + ".n.bias"] - st1[:, 0:1] * st1[:, 1:2] * sd[p + ".n.weight"]
            e = max(e, ((rb[idx].to(F64) - shift).abs() / (shift.abs() + (st1[:, 0:1] * st1[:, 1:2] * sd[p + ".n.weight"]).abs())).max().item())
            print(f"{w} stack {i} norm2_fold F={Fn}: max relative error of rstd0 rstd1 / res_scale / res_shift {e:.2e} (bound {FOLD_REL:.0e})")
            assert e <= FOLD_REL
            hb, hmid = guarded_zp(Fn, H, W, Cc)
            pb = conv_part_buf(Fn, H, W, Cc)
            check_plan(s, f"stack {i} block conv", Fn)
            res = {}

            def conv0():
                refill(hb, pb)
                res["mrh"] = conv_call(y1, Wb0, H, W, hmid, pb.t, mr=mrE, Ef=Ef, relu=1)
                return [digest(hmid), pb.t.clone()], [yb, hb, pb] + bufs

            _run_twice(f"{w} stack {i} block 0 conv0 (Ef) {H}x{W}x{Cc} F={Fn}", conv0)
            mrh = res["mrh"]
            assert all_finite(hmid) and pads_zero(hmid) and all_finite(pb.t)
            ref_h, _ = Rf.block(y1[idx], sd, p + ".blocks.0", n=p + ".n")
            check_frames(f"{w} stack {i} block 0 conv0 F={Fn}", hmid, ref_h, idx, CONV_FLOOR)
            check_stats(f"{w} stack {i} block 0 conv0 (mean, rstd) F={Fn}", mrh[idx], Rf.stats(hmid[idx], zp=True))
            del pb
            ob, out = guarded_zp(Fn, H, W, Cc)
            pb = conv_part_buf(Fn, H, W, Cc)

            def conv1():
                refill(ob, pb)
                res["mr"] = conv_call(hmid, Wb1, H, W, out, pb.t, mr=mrh, S1=S1, S2=S2, relu=1, residual=y1, rs=rs, rb=rb)
                return [digest(out), pb.t.clone()], [yb, hb, ob, pb] + bufs

            _run_twice(f"{w} stack {i} block 0 conv1 (affine residual) F={Fn}", conv1)
            assert all_finite(out) and pads_zero(out) and all_finite(pb.t)
            ref = Rf.nhwc(x0) + Rf.conv(hmid[idx], sd, p + ".blocks.0.conv1")
            check_frames(f"{w} stack {i} block 0 conv1 F={Fn}", out, ref, idx, CONV_FLOOR)
            check_stats(f"{w} stack {i} block 0 (mean, rstd) F={Fn}", res["mr"][idx], Rf.stats(out[idx], zp=True))
            del yb, y1, hb, hmid, ob, out, pb, bufs, mrE, Ef, rs, rb, chan


def test_block1_and_the_training_layout(model):
    """block 1 (and every block of the training layout): conv0 with S1 / S2, conv1 with residual (the last stack writes through `out=`
    into a slice of a larger NaN-filled buffer, as `_forward_impl` does with cnn_out[f0:f0+F]); the training layout's vpt_affine_norm_zp and
    vpt_add_stats (add_zp) beside it"""
    w, s, pol, sd, prep = model
    last_stack = len(s["stacks"]) - 1
    for i, sh in enumerate(s["stacks"]):
        H, W, Cc = sh["H"] // 2, sh["W"] // 2, sh["C"]
        st = prep.stacks[i]
        p = f"img_process.cnn.stacks.{i}"
        for Fn in chunks(s):
            xb, x = guarded_zp(Fn, H, W, Cc)
            fill(x, 300 + i)
            idx = sel_frames(Fn)
            mr = in_chunks(lambda v: Rf.stats(v, zp=True), x).float()
            # training layout: x0 = n(y1) as a pass (here: n(x)), the residual add as a pass below (x + r, r = the branch output)
            per = (H + 1) * (W + 1) * Cc
            P = lib().vpt_norm_stat_parts((H + 1) * (W + 1), Cc)
            nb, pn = Guarded(Fn * per, BF16), Guarded(Fn * P * 2)
            xn = nb.t.view(Fn, H + 1, W + 1, Cc)

            def affine():
                refill(nb, pn)
                nat.check(lib().vpt_affine_norm_zp(x.data_ptr(), mr.data_ptr(), st["n_g"].data_ptr(), st["n_b"].data_ptr(), xn.data_ptr(), pn.ptr(),
                                                   Fn, H, W, Cc, stream()), "vpt_affine_norm_zp")
                return [digest(xn), pn.t.clone()], [xb, nb, pn]

            _run_twice(f"{w} stack {i} affine_norm_zp F={Fn}", affine)
            assert all_finite(xn) and pads_zero(xn) and all_finite(pn.t)
            ref = Rf.nhwc(F.group_norm(Rf.nchw(x[idx]), 1, sd[p + ".n.weight"], sd[p + ".n.bias"], eps=1e-5))
            check_frames(f"{w} stack {i} affine_norm_zp F={Fn}", xn, ref, idx, CONV_FLOOR)
            mr0 = ops.stats_finalize(pn.t.view(Fn, P, 2), Fn, P, H * W * Cc)
            check_stats(f"{w} stack {i} affine_norm_zp (mean, rstd) F={Fn}", mr0[idx], Rf.stats(xn[idx], zp=True))
            del nb, xn, pn
            Wb, S1, S2 = st["convs"][2]
            hb, hmid = guarded_zp(Fn, H, W, Cc)
            pb = conv_part_buf(Fn, H, W, Cc)
            check_plan(s, f"stack {i} block conv", Fn)
            res = {}

            def conv0():
                refill(hb, pb)
                res["mrh"] = conv_call(x, Wb, H, W, hmid, pb.t, mr=mr, S1=S1, S2=S2, relu=1)
                return [digest(hmid), pb.t.clone()], [xb, hb, pb]

            _run_twice(f"{w} stack {i} block 1 conv0 {H}x{W}x{Cc} F={Fn}", conv0)
            assert all_finite(hmid) and pads_zero(hmid) and all_finite(pb.t)
            ref_h, _ = Rf.block(x[idx], sd, p + ".blocks.1")
            check_frames(f"{w} stack {i} block 1 conv0 F={Fn}", hmid, ref_h, idx, CONV_FLOOR)
            check_stats(f"{w} stack {i} block 1 conv0 (mean, rstd) F={Fn}", res["mrh"][idx], Rf.stats(hmid[idx], zp=True))
            del pb
            Wb, S1, S2 = st["convs"][3]
            ob = Guarded((Fn + 2) * per, BF16)  # the last stack writes frames 1 .. F of it
            big = ob.t.view(Fn + 2, H + 1, W + 1, Cc)
            out = big[1:Fn + 1]
            pb = conv_part_buf(Fn, H, W, Cc)

            def conv1():
                refill(ob, pb)
                res["mr"] = conv_call(hmid, Wb, H, W, out, pb.t, mr=res["mrh"], S1=S1, S2=S2, relu=1, residual=x)
                assert (big[0].view(torch.int16) == -1).all() and (big[Fn + 1].view(torch.int16) == -1).all(), "wrote outside its chunk's frames"
                return [digest(out), pb.t.clone()], [xb, hb, ob, pb]

            _run_twice(f"{w} stack {i} block 1 conv1 (residual{', out= slice' if i == last_stack else ''}) F={Fn}", conv1)
            assert all_finite(out) and pads_zero(out) and all_finite(pb.t)
            ref = x[idx][:, :-1, :-1].to(F64) + Rf.conv(hmid[idx], sd, p + ".blocks.1.conv1")
            check_frames(f"{w} stack {i} block 1 conv1 F={Fn}", out, ref, idx, CONV_FLOOR)
            check_stats(f"{w} stack {i} block 1 (mean, rstd) F={Fn}", res["mr"][idx], Rf.stats(out[idx], zp=True))
            P = lib().vpt_add_stat_parts(per)
            pa = Guarded(Fn * P * 2)

            def add():
                refill(ob, pa)
                nat.check(lib().vpt_add_stats(x.data_ptr(), hmid.data_ptr(), out.data_ptr(), pa.ptr(), Fn, per, stream()), "vpt_add_stats")
                assert (big[0].view(torch.int16) == -1).all() and (big[Fn + 1].view(torch.int16) == -1).all(), "wrote outside its chunk's frames"
                return [digest(out), pa.t.clone()], [xb, hb, ob, pa]

            _run_twice(f"{w} stack {i} add_zp F={Fn}", add)
            assert all_finite(out) and pads_zero(out) and all_finite(pa.t)
            bad = (out[idx] != (x[idx].to(F64) + hmid[idx].to(F64)).to(BF16)).sum().item()
            print(f"{w} stack {i} add_zp F={Fn}: mismatches against float64 x + r rounded once {bad} (bound 0)")
            assert bad == 0
            mra = ops.stats_finalize(pa.t.view(Fn, P, 2), Fn, P, H * W * Cc)
            check_stats(f"{w} stack {i} add_zp (mean, rstd) F={Fn}", mra[idx], Rf.stats(out[idx], zp=True))
            del xb, x, hb, hmid, ob, big, out, pb, pa


def test_idm_conv3d_pre_stage(model):
    """vpt_conv3d_t5 at B x T = 4 x 128 (and 2 x 128, and one sequence of each small count), 128 x 128 px, C = 128 against float64 conv3d_stage, on the frames at both ends of
    every sequence (the clipped time window) and one in the middle"""
    w, s, pol, sd, prep = model
    if s["conv3d"] is None:
        pytest.skip("the policies have no conv3d pre-stage")
    H, W, _ = s["cfg"].img_shape
    Cc, T = s["conv3d"], s["t"]
    w3, b3 = prep.conv3d
    for Fn in chunks(s):
        B, T = (Fn // s["t"], s["t"]) if Fn % s["t"] == 0 else (1, Fn)  # a few frames: one short sequence
        img = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=torch.Generator(device=DEV).manual_seed(Fn), device=DEV)
        img[-1, -3:] = 100 + img[-1, -3:] // 32  # nearly flat last frames
        P = lib().vpt_conv3d_stat_parts(H, W, Cc)
        ob, out = guarded_zp(Fn, H, W, Cc)
        pb = Guarded(Fn * P * 2)

        def call():
            refill(ob, pb)
            nat.check(lib().vpt_conv3d_t5(img.data_ptr(), w3.data_ptr(), b3.data_ptr(), out.data_ptr(), pb.ptr(), B, T, H, W, Cc, 0, stream()),
                      "vpt_conv3d_t5")
            return [digest(out), pb.t.clone()], [ob, pb]

        _run_twice(f"{w} conv3d_t5 B={B} T={T} F={Fn}", call)
        assert all_finite(out) and pads_zero(out) and all_finite(pb.t)
        mr = ops.stats_finalize(pb.t.view(Fn, P, 2), Fn, P, H * W * Cc)
        got, ref, fr = [], [], []
        for b in range(B):
            for t in sorted({t for t in (0, 1, T // 2, T - 2, T - 1) if 0 <= t < T}):
                lo, hi = max(0, t - 2), min(T, t + 3)
                ref.append(Rf.conv3d(img[b:b + 1, lo:hi], sd, "conv3d_layer")[t - lo])
                fr.append(b * T + t)
        ref = torch.stack(ref)
        check_bf16(f"{w} conv3d_t5 F={Fn} (sequence ends and middles)", out[fr][:, :-1, :-1], ref, CONV_FLOOR)
        check_stats(f"{w} conv3d_t5 (mean, rstd) F={Fn}", mr[fr], Rf.stats(out[fr], zp=True))
        del ob, out, pb, img


# ---------------------------------------------------------------------------------------------------------------------
# linear folds, heads
# ---------------------------------------------------------------------------------------------------------------------
def edge_rows(M, K, seed):
    """bf16 rows: randn, odd rows relu(randn) + 3, the last row 3 + randn * 3/64 (M = 1: the DC row)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn((M, K), generator=g, device=DEV)
    x[1::2] = x[1::2].relu() + 3.0
    if M > 1:
        x[-1] = 3.0 + x[-1] * (3.0 / 64)
    else:
        x[0] = x[0].relu() + 3.0
    return x.to(BF16)


def guarded_rows(M, N, dtype=BF16, ld=None):
    b = Guarded(M * (ld or N), dtype)
    return b, b.t.view(M, ld or N)


ROWS = [2048, 1096, 64, 9, 8, 3, 1]  # the tensor-core kernel from 9 rows (partial M tiles but at 2048), weight streaming up to 8


def check_gemm_plan(name, M, part):
    """the GEMM kernel a call of M rows ran, read from the statistics partials [M][P][2] (P >= 2) it wrote with stat_mode=1: the
    weight-streaming kernel's row pass puts each row's whole (sum, sumsq) in slot 0 and zeros in the others, the tensor-core kernel one
    partial per 64-column half of its N tiles.  It must be the weight-streaming kernel up to 8 rows and the tensor-core kernel above."""
    assert part.shape[1] >= 2
    streamed = bool((part[:, 1:] == 0).all())
    print(f"{name}: {'gemv_small_kernel' if streamed else 'gemm_tc_kernel'} ({part.shape[1]} partials per row)")
    assert streamed == (M <= 8), name


def plan_partials(x, Wb, M, N, K, **kw):
    """The statistics partials of a sibling of a GEMM call that writes none (the heads, the fused QKVR): the same x, weights, M, N and K
    into a scratch output, with stat_mode=1 partials and without destination segments.  vpt_gemm_bf16 picks its kernel by M and K alone
    for such calls (csrc/gemv_small.cuh, `try_launch_gemv_small`), so the sibling runs the call's kernel (`check_gemm_plan`)."""
    P = ops.gemm_stat_parts(N)
    ld = kw.pop("ld_out", N)
    out = torch.empty((M, ld), dtype=F32, device=DEV)
    part = torch.empty((M, P, 2), dtype=F32, device=DEV)
    ops.gemm(x, Wb, out, M, N, K, ld_out=ld, stat_part=part, stat_mode=1, **kw)
    torch.cuda.synchronize()
    nat.device_check()
    return part


def _linear_case(name, x, fold, N, ref, *, mr=None, relu=0, residual=None, flat_floor=LIN_FLOOR):
    """one vpt_gemm_bf16 call with stat_mode=1 partials into guarded buffers: run twice, output against `ref`, statistics against float64
    LayerNorm statistics of the stored output, and the kernel it ran (`check_gemm_plan`)"""
    M, K = x.shape
    Wb, S1, S2 = fold
    P = ops.gemm_stat_parts(N)
    ob, out = guarded_rows(M, N)
    pb = Guarded(M * P * 2)
    xb, xg = guarded_rows(M, K)
    xg.copy_(x)
    res = {}

    def call():
        refill(ob, pb)
        ops.gemm(xg, Wb, out, M, N, K, mr=mr, S1=S1 if mr is not None else None, S2=S2, relu=relu, residual=residual,
                 stat_part=pb.t, stat_mode=1)
        res["mr"] = ops.stats_finalize(pb.t, M, P, N)
        return [out.clone(), pb.t.clone()], [ob, pb, xb]

    _run_twice(name, call)
    assert all_finite(out) and all_finite(pb.t)
    check_gemm_plan(name, M, pb.t.view(M, P, 2))
    kinds = ["const" if (r == M - 1 and M > 1) else "dc" if (r % 2 == 1 or M == 1) else "randn" for r in range(M)]
    for k in dict.fromkeys(kinds):
        j = [r for r in range(M) if kinds[r] == k]
        check_bf16(f"{name} [{k} rows]", out[j], ref[j], flat_floor if k == "const" else LIN_FLOOR)
    check_stats(f"{name} (mean, rstd)", res["mr"], Rf.stats(out))


@pytest.mark.parametrize("M", ROWS)
def test_linear_folds(model, M):
    """dense (ZP rows, zero weight columns at the pads), linear, mlp0 (LayerNorm fold, ReLU), mlp1 (residual; relu=2 on the last block),
    proj (residual = x_hat) and lastlayer through vpt_gemm_bf16 against float64 fanin_linear / F.linear: M = 2048 on the tensor-core
    kernel, M = 1096, 64 and 9 on its partial M tiles (many-environment rollouts), M = 1, 3 and 8 on the small-M streaming kernel"""
    w, s, pol, sd, prep = model
    cfg = s["cfg"]
    Hf, Wf, C2, kd = s["dense"]
    h = s["h"]
    L = len(prep.layers) - 1
    b = f"recurrent_layer.blocks.{L}"
    xz = torch.zeros((M, Hf + 1, Wf + 1, C2), dtype=BF16, device=DEV)
    xz[:, :-1, :-1] = edge_rows(M, Hf * Wf * C2, 1).view(M, Hf, Wf, C2)
    xd = xz.view(M, kd)
    mr = Rf.stats(xz, zp=True).float()
    _linear_case(f"{w} dense {kd}->{cfg.cnn_outsize} M={M}", xd, prep.dense, cfg.cnn_outsize,
                 Rf.linear(_dense_from_zp(xd, cfg), sd, "img_process.cnn.dense"), mr=mr, relu=1, flat_floor=DENSE_FLAT_FLOOR if M > 8 else LIN_FLOOR)
    x = edge_rows(M, cfg.cnn_outsize, 2)
    _linear_case(f"{w} linear M={M}", x, prep.linear, h, Rf.linear(x, sd, "img_process.linear"), mr=Rf.stats(x).float(), relu=1)
    y = edge_rows(M, h, 3)
    mr = Rf.stats(y).float()
    _linear_case(f"{w} mlp0 M={M}", y, prep.layers[L]["mlp0"], 4 * h, Rf.linear(y, sd, b + ".mlp0"), mr=mr, relu=1)
    a = edge_rows(M, 4 * h, 4)
    ref = y.to(F64) + Rf.linear(a, sd, b + ".mlp1", relu=False)
    _linear_case(f"{w} mlp1 (last block, relu=2) M={M}", a, prep.layers[L]["mlp1"], h, ref.relu(), relu=2, residual=y)
    _linear_case(f"{w} mlp1 M={M}", a, prep.layers[L]["mlp1"], h, ref, residual=y)
    a = edge_rows(M, h, 5)
    ref = y.to(F64) + Rf.plain_linear(a, sd, b + ".r.orc_block.proj_layer")
    _linear_case(f"{w} proj M={M}", a, prep.layers[L]["proj"], h, ref, residual=y)
    if "lastlayer" in s["linears"]:
        z = edge_rows(M, h, 6).relu()
        _linear_case(f"{w} lastlayer M={M}", z, prep.last, h, Rf.linear(z, sd, "lastlayer"), mr=Rf.stats(z).float(), relu=1)
    nat.device_check()


@pytest.mark.parametrize("M", ROWS)
def test_heads_and_log_softmax(model, M):
    """the heads GEMM (out_scale = 1 / temperature, fp32 out, ragged N, ld > N: the columns beyond N stay NaN) against float64
    F.linear / temperature, then vpt_log_softmax of every head (each of the IDM's sub-actions) reading the raw logits between NaN guard
    bands and columns, against float64 log_softmax of the stored logits"""
    w, s, pol, sd, prep = model
    hp = pol._heads_prepared()
    N, ld, temp = s["ntot"], s["ld_logits"], pol.temperature
    assert hp["ntot"] == N and ld > N
    lat = edge_rows(M, s["h"], 7)
    Wt = torch.cat([getattr(pol.pi_head, name).linear_layer.weight for name, *_ in s["head_cols"]]).to(F64)
    bias = torch.cat([getattr(pol.pi_head, name).linear_layer.bias for name, *_ in s["head_cols"]]).to(F64)
    ref = (lat.to(F64) @ Wt.T + bias) / temp
    scale = (lat.to(F64).abs() @ Wt.abs().T + bias.abs()) / temp
    rb, raw = guarded_rows(M, N, F32, ld=ld)
    Wb, _, S2 = hp["pi"]

    def heads():
        refill(rb)
        ops.gemm(lat, Wb, raw, M, N, s["h"], S2=S2, out_scale=1.0 / temp, ld_out=ld)
        assert (raw[:, N:].view(torch.int32) == -1).all(), "heads GEMM wrote beyond its N columns"
        return [raw[:, :N].clone()], [rb]

    _run_twice(f"{w} heads GEMM M={M} N={N} ld={ld}", heads)
    check_gemm_plan(f"{w} heads GEMM M={M}", M, plan_partials(lat, Wb, M, N, s["h"], S2=S2, out_scale=1.0 / temp, ld_out=ld))
    assert all_finite(raw[:, :N])
    check_sum(f"{w} heads logits M={M}", raw[:, :N], ref, scale, HEAD_ELEM, HEAD_L2)
    for name, c0, n, cnt in s["head_cols"]:
        assert hp["cols"][name] == (c0, n * cnt)
        for k in range(cnt):
            lb, lp = guarded_rows(M, n, F32)

            def lsm():
                refill(lb)
                nat.check(lib().vpt_log_softmax(raw.data_ptr(), ld, c0 + k * n, n, lp.data_ptr(), M, stream()), "vpt_log_softmax")
                return [lp.clone()], [rb, lb]

            _run_twice(f"{w} log_softmax {name}[{k}] n={n} M={M}", lsm)
            e = (lp.to(F64) - torch.log_softmax(raw[:, c0 + k * n:c0 + (k + 1) * n].to(F64), -1)).abs().max().item()
            if k == 0:
                print(f"{w} log_softmax {name} n={n} M={M}: max |err| {e:.2e} (bound {LOGSM_ABS:.0e})")
            assert torch.isfinite(lp).all() and e <= LOGSM_ABS


# ---------------------------------------------------------------------------------------------------------------------
# attention block: fused QKVR, KV memory copies, attention
# ---------------------------------------------------------------------------------------------------------------------
def test_fused_qkvr(model):
    """the Q | K | V | R GEMM with column segments (policy.py, `_block`) at B = 16 (IDM: 4), t = 128, and for the policies at the
    rollout rows (B, t) = (1, 1), (8, 1) (the weight-streaming kernel), (9, 1) and (64, 1) (partial M tiles), each in the pytree layout
    and the ring layout: K / V land in the rows of full_k / full_v after the memory rows (untouched, NaN), or in (B, 1, h) step rows for
    the ring (`seg` the identity); R in fp32 with a row pitch wider than its columns (untouched, NaN); against four float64 F.linear"""
    w, s, pol, sd, prep = model
    h, heads, maxlen = s["h"], s["heads"], s["maxlen"]
    o = "recurrent_layer.blocks.0.r.orc_block"
    Wc, _, bc = prep.layers[0]["qkvr"]
    assert Wc.shape[0] == s["qkvr"]
    nr = NBASIS * heads if s["causal"] else 0
    ldr = nr + 8
    cases = [(4 if s["conv3d"] else 16, s["t"], "pytree")]
    if s["causal"]:
        cases += [(B, 1, layout) for B in (1, 8, 9, 64) for layout in ("pytree", "ring")]
    for B, t, layout in cases:
        M = B * t
        mem = maxlen if layout == "pytree" else 0  # memory rows before the step's K / V rows
        T = mem + t
        name = f"{w} fused qkvr B={B} t={t} {layout} layout"
        xhat = edge_rows(M, h, 8 if t > 1 else 8 + M)
        qb, q = guarded_rows(M, h)
        kb, vb = Guarded(B * T * h, BF16), Guarded(B * T * h, BF16)
        fk, fv = kb.t.view(B, T, h), vb.t.view(B, T, h)
        Rb, R = guarded_rows(M, ldr, F32)
        dsts = [(0, q, h, False), (h, fk, h, True), (2 * h, fv, h, True)] + ([(3 * h, R, ldr, False)] if nr else [])

        def call():
            refill(qb, kb, vb, Rb)
            ops.gemm(xhat, Wc, q, M, Wc.shape[0], h, S2=bc, seg=(t, T, mem), dsts=dsts)
            for full in (fk, fv):
                assert (full[:, :mem].view(torch.int16) == -1).all(), "wrote into the memory rows"
            assert (R[:, nr:].view(torch.int32) == -1).all(), "wrote beyond the R columns"
            return [q.clone(), fk[:, mem:].clone(), fv[:, mem:].clone(), R[:, :nr].clone()], [qb, kb, vb, Rb]

        _run_twice(name, call)
        check_gemm_plan(name, M, plan_partials(xhat, Wc, M, Wc.shape[0], h, S2=bc))
        refs = [Rf.plain_linear(xhat, sd, o + ".q_layer"), Rf.plain_linear(xhat, sd, o + ".k_layer", bias=False),
                Rf.plain_linear(xhat, sd, o + ".v_layer", bias=False)]
        for c, got, ref in zip("qkv", (q, fk[:, mem:].reshape(M, h), fv[:, mem:].reshape(M, h)), refs):
            check_bf16(f"{name} {c}", got, ref, LIN_FLOOR)
        if nr:
            ref = Rf.plain_linear(xhat, sd, o + ".r_layer")
            Wr = sd[o + ".r_layer.weight"]
            check_sum(f"{name} R (fp32)", R[:, :nr], ref, xhat.to(F64).abs() @ Wr.abs().T + sd[o + ".r_layer.bias"].abs(), HEAD_ELEM, HEAD_L2)
        del qb, kb, vb, Rb, q, fk, fv, R


def test_copy_rows2(model):
    """the KV memory into `full` (fp32 state -> bf16) and out of it (bf16 -> fp32 state) at B = 16: bit-exact with slicing + .to(dtype);
    the source sits between NaN guard bands, the destination rows outside the copy stay NaN"""
    w, s, pol, sd, prep = model
    if not s["causal"]:
        pytest.skip("the IDM has no KV memory")
    h, maxlen, t, B = s["h"], s["maxlen"], s["t"], 16
    T = maxlen + t
    g = torch.Generator(device=DEV).manual_seed(9)
    mb = [Guarded(B * maxlen * h) for _ in range(2)]
    mem = [b.t.view(B, maxlen, h) for b in mb]
    for m in mem:
        m.copy_(torch.randn((B, maxlen, h), generator=g, device=DEV))
    fb = [Guarded(B * T * h, BF16) for _ in range(2)]
    full = [b.t.view(B, T, h) for b in fb]

    def load():
        refill(*fb)
        ops.copy_rows2(mem[0], mem[1], 0, full[0], full[1], 0, maxlen)
        return [f.clone() for f in full], mb + fb

    _run_twice(f"{w} copy_rows2 memory -> full", load)
    for m, f in zip(mem, full):
        assert torch.equal(f[:, :maxlen], m.to(BF16)) and (f[:, maxlen:].view(torch.int16) == -1).all()
    for f in full:
        f[:, maxlen:] = torch.randn((B, t, h), generator=g, device=DEV).to(BF16)
    nb = [Guarded(B * maxlen * h) for _ in range(2)]
    new = [b.t.view(B, maxlen, h) for b in nb]

    def store():
        refill(*nb)
        ops.copy_rows2(full[0], full[1], T - maxlen, new[0], new[1], 0, maxlen)
        return [n.clone() for n in new], fb + nb

    _run_twice(f"{w} copy_rows2 full -> state", store)
    for f, n in zip(full, new):
        assert torch.equal(n, f[:, T - maxlen:].float())
    print(f"{w} copy_rows2 B={B} maxlen={maxlen} h={h}: bit-exact both ways (bound 0)")


@pytest.mark.parametrize("t", [128, 1])
def test_attention(model, t):
    """vpt_attention at the model's heads, maxlen = 128, B = 16 (policies: clipped causal with the relative-position term; one row with
    `first` set over a zero state mask -- its memory fully masked -- and the rest with a random state mask) and the IDM's unmasked attention
    at t = 128, B = 4; q, full_k, full_v, R between NaN guard bands; against float64"""
    w, s, pol, sd, prep = model
    h, heads = s["h"], s["heads"]
    causal = s["causal"]
    if not causal and t != 128:
        pytest.skip("the IDM runs whole 128-frame chunks")
    maxlen = s["maxlen"]
    B = 16 if causal else 4
    T = maxlen + t
    g = torch.Generator(device=DEV).manual_seed(10 + t)
    bufs = dict(Q=Guarded(B * t * h, BF16), Kf=Guarded(B * T * h, BF16), Vf=Guarded(B * T * h, BF16))
    x = dict(Q=bufs["Q"].t.view(B * t, h), Kf=bufs["Kf"].t.view(B, T, h), Vf=bufs["Vf"].t.view(B, T, h))
    x["Q"].copy_(torch.randn((B * t, h), generator=g, device=DEV) * 3)
    x["Kf"].copy_(torch.randn((B, T, h), generator=g, device=DEV) * 3)
    x["Vf"].copy_(torch.randn((B, T, h), generator=g, device=DEV))
    ld_r = 0
    if causal:
        bufs["R"] = Guarded(B * t * NBASIS * heads)
        x["R"] = bufs["R"].t.view(B * t, NBASIS * heads)
        x["R"].copy_(torch.randn((B * t, NBASIS * heads), generator=g, device=DEV))
        ld_r = NBASIS * heads
        x["b_nd"] = sd["recurrent_layer.blocks.0.r.orc_block.b_nd"].float().contiguous()
        first = torch.zeros(B, t, dtype=torch.uint8, device=DEV)
        first[3, 0] = 1
        smask = (torch.rand((B, maxlen), generator=g, device=DEV) > 0.3).to(torch.uint8)
        smask[3] = 0
        x["first_u8"], x["smask_u8"] = first, smask
    ob, out = guarded_rows(B * t, h)

    def call():
        refill(ob)
        nat.check(lib().vpt_attention(x["Q"].data_ptr(), x["Kf"].data_ptr(), x["Vf"].data_ptr(), _p(x.get("R")), ld_r, _p(x.get("b_nd")),
                                      _p(x.get("first_u8")), t if causal else 0, _p(x.get("smask_u8")), out.data_ptr(), B, t, maxlen, heads,
                                      NBASIS if causal else 0, int(causal), stream()), "vpt_attention")
        return [out.clone()], list(bufs.values()) + [ob]

    _run_twice(f"{w} attention heads={heads} t={t} maxlen={maxlen} B={B}", call)
    if causal:
        ref = attention_ref(x, B, t, maxlen, heads)
    else:
        D = h // heads
        q = x["Q"].to(F64).reshape(B, t, heads, D).transpose(1, 2)
        k = x["Kf"].to(F64).reshape(B, t, heads, D).transpose(1, 2)
        v = x["Vf"].to(F64).reshape(B, t, heads, D).transpose(1, 2)
        ref = (torch.softmax(q @ k.transpose(-1, -2) / D, -1) @ v).transpose(1, 2).reshape(B * t, h)
    check_bf16(f"{w} attention heads={heads} t={t}", out, ref, ATTN_FLOOR)
    if causal:
        check_bf16(f"{w} attention heads={heads} t={t} [row with its memory fully masked]", out[3 * t:4 * t], ref[3 * t:4 * t], ATTN_FLOOR)
    if causal and t == 1:
        _ring_rows_case(w, x, out, B, maxlen, heads, g)


def _ring_rows_case(w, x, lin_out, B, maxlen, heads, g):
    """The same step on a ring (`vpt_ring_write_rows`, then `vpt_attention_ring_rows`) at a random `off`, random per-environment
    `row_off` and batch rows mapped to a permutation of E = B + 3 environments, three of them inert (-1): every other row equals the
    linear layout's row bit for bit, inert rows are zero, and environments no row lists keep every byte."""
    h = x["Q"].shape[1]
    E = B + 3
    rows = torch.randperm(E, generator=torch.Generator().manual_seed(11))[:B].to(torch.int32)
    rows[[2, 7, B - 1]] = -1
    off = torch.randint(0, maxlen, (1,), generator=g, device=DEV, dtype=torch.int32)
    row_off = torch.randint(0, maxlen, (E,), generator=g, device=DEV, dtype=torch.int32)
    kb, vb, mb = Guarded(E * maxlen * h, BF16), Guarded(E * maxlen * h, BF16), Guarded(E * maxlen, torch.uint8)
    kr, vr, mask = kb.t.view(E, maxlen, h), vb.t.view(E, maxlen, h), mb.t.view(E, maxlen)
    rows_d = rows.to(DEV)
    # memory key j of the batch row b listed at ring row r sits at (off + row_off[r] + j) % maxlen; unlisted rows hold randn
    k0 = torch.randn((E, maxlen, h), generator=g, device=DEV).to(BF16)
    v0 = torch.randn((E, maxlen, h), generator=g, device=DEV).to(BF16)
    m0 = (torch.rand((E, maxlen), generator=g, device=DEV) > 0.5).to(torch.uint8)
    for b in range(B):
        r = int(rows[b])
        if r >= 0:
            slot = (off + row_off[r] + torch.arange(maxlen, device=DEV)) % maxlen
            k0[r, slot], v0[r, slot], m0[r, slot] = x["Kf"][b, :maxlen], x["Vf"][b, :maxlen], x["smask_u8"][b]
    k_new, v_new = x["Kf"][:, maxlen].contiguous(), x["Vf"][:, maxlen].contiguous()
    ob = Guarded(B * h, BF16)

    def call():
        kr.copy_(k0)
        vr.copy_(v0)
        mask.copy_(m0)
        ob.raw.fill_(0xFF)
        ops_ring.ring_write(k_new, v_new, kr, vr, mask, off, x["first_u8"], rows=rows_d, row_off=row_off)
        nat.check(lib().vpt_attention_ring_rows(x["Q"].data_ptr(), kr.data_ptr(), vr.data_ptr(), x["R"].data_ptr(), x["R"].stride(0),
                                                x["b_nd"].data_ptr(), x["first_u8"].data_ptr(), x["first_u8"].stride(0), mask.data_ptr(),
                                                off.data_ptr(), rows_d.data_ptr(), row_off.data_ptr(), ob.ptr(), B, maxlen, heads,
                                                x["b_nd"].shape[0], stream()), "vpt_attention_ring_rows")
        return [ob.t.clone(), kr.clone(), vr.clone(), mask.clone()], [kb, vb, mb, ob]

    _run_twice(f"{w} attention_ring_rows heads={heads} B={B} E={E}", call)
    out = ob.t.view(B, h)
    real = rows >= 0
    bad = (out[real] != lin_out[real]).sum().item()
    print(f"{w} attention_ring_rows heads={heads} B={B} E={E}: mismatches against the linear layout {bad}, "
          f"nonzero values in the {int((~real).sum())} inert rows {int((out[~real] != 0).sum())} (bound 0)")
    assert bad == 0 and bool((out[~real] == 0).all())
    unlisted = sorted(set(range(E)) - set(rows[real].tolist()))
    assert unlisted and all(torch.equal(a[unlisted], b[unlisted]) for a, b in ((kr, k0), (vr, v0), (mask, m0))), "an unlisted environment changed"
