"""Kernels of the fp32-parity mode (`policy.set_precision("fp32")`, video-pre-training_b200/precise.py, csrc/precise.cuh) at the shapes the
released models run (1x / 2x / 3x widths and the 4x IDM), each on isolated fp32 inputs, against the float64 unfused layers of
tests/fwd_refs.py (the oracle's GroupNorm -> conv -> ReLU, LayerNorm -> linear, max-pool, attention).  The kernels get the weights of the
product's own `prepared_precise()` / `_heads_prepared_precise()`, so the weight preparation (`_split_w`, the OIHW -> [Cout][tap][Cin] conv
layout, the dense layer's C,H,W -> H,W,C permutation, `fc_w / 255`) is under test with the kernels.  Each reference is computed from the
same fp32 inputs, not from the hi / lo splits, so the split error is part of what is measured.

Every call also keeps the buffer contract: outputs, the (mean, rstd) table, the hi / lo splits and the running sum `acc` of `gemm3` start as
NaN between NaN guard bands; every element of [M][N] comes back finite and the guards untouched (the pad columns N .. ld of an output are
not part of the contract); the inputs sit between NaN guards too; two identical calls give identical bits (large outputs are compared
through a position-weighted digest).

Inputs hold three kinds of frame or row: randn, a mean six times the spread, and a spread 1/64 of the mean (where a norm's statistics
cancel most of their bits).  The conv and linear units compare the first, the last and three rows or frames between, which hold every
kind; each check prints, per kind, the worst rel-L2 of a row or frame and the worst max |err| / rms(ref) of one beside its bound, and
each test prints its peak device memory."""
import gc

import pytest
import torch
import torch.nn.functional as F

import fwd_refs as Rf
import test_gpu_forward_shapes as FS
from test_gpu_backward_shapes import Guarded, _run_twice
from test_gpu_long_attention import fwd_ref as attention_ref
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import precise as P

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U8 = torch.uint8
SHAPES = {w: Rf.forward_shapes(w) for w in Rf.MODELS}

# Bounds: each is at most 4x the worst value measured on an H100 80GB HBM3 (SXM, 700 W power limit), given beside it: the rel-L2 of a
# checked row / frame and its max |err| / rms(ref).  A dropped hi / lo launch or a wrong split costs ~2^-9 = 2e-3 of a layer's output.
CONV_L2, CONV_MAX = 3e-5, 2.5e-4  # the normalised convs: GroupNorm -> 3 hi / lo launches -> ReLU; measured 7.5e-6, 6.1e-5
FC_L2, FC_MAX = 2.2e-5, 1.6e-4    # firstconv_pool and conv3d_t5 with fp32 output; measured 5.5e-6, 3.9e-5
NORM_L2, NORM_MAX = 2e-5, 2.5e-5  # the post-pool GroupNorm; measured 4.7e-6, 6.1e-6 (the fp32 mean of a near-constant frame)
# linear layers through gemm3: the small-M kernel (M <= 8) and the tensor cores at K <= 4096 measured 6.6e-6, 4.1e-5.  On the tensor
# cores the error grows in proportion to K -- the wgmma fp32 accumulation (the dense layer, K = 32 768 .. 131 072: rel-L2 1.25e-9 K,
# max 6.5e-9 K; mlp1, K = 4h: the same slope) -- so their bound adds a term per K
LIN_L2, LIN_MAX = 2.6e-5, 1.6e-4
TC_L2_PER_K, TC_MAX_PER_K = 5e-9, 2.6e-8
VALUE_REL = 3e-4                  # the value head, one output per row: relative error of it; measured 7.4e-5
ATTN_L2, ATTN_MAX = 8e-6, 4e-5    # vpt_attention_f32; measured 1.9e-6, 9.4e-6
STAT_MEAN, STAT_RSTD = 2e-5, 2.5e-7  # group_stats_f32 vs float64 of its input: |d mean| * rstd, |d rstd| / rstd; measured 4.7e-6, 6.0e-8


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
    """(width, shapes, policy on the device, float64 net state dict on the device, prepared_precise()); one model at a time"""
    w = request.param
    pol, sd = Rf.make_model(w)
    pol = pol.to(DEV).set_precision("fp32")
    m = [w, SHAPES[w], pol, Rf.SD64(sd, DEV), pol.net.prepared_precise()]
    yield m
    # prepared_precise() is one more weight-layout cache a policy holds through bound methods of itself: a reference cycle, which only
    # the cyclic collector frees.  pytest still holds the yielded value here, so it is emptied before collecting
    m.clear()
    del pol, sd
    FS._WEIGHTS.clear()
    gc.collect()
    torch.cuda.empty_cache()
    print(f"{w} model released: {torch.cuda.memory_allocated() / 2 ** 30:.2f} GiB still allocated")


@pytest.fixture(autouse=True)
def peak_memory(request):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"{request.node.name}: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


frame_kind, refill, all_finite, digest = FS.frame_kind, FS.refill, FS.all_finite, FS.digest


def sel_frames(Fn):
    """the checked frames / rows: the first, the last and three between (all of them when there are fewer)"""
    return sorted({f for f in (0, 1, Fn // 2, Fn - 2, Fn - 1) if 0 <= f < Fn})


def fill32(t, seed, relu=False):
    """fp32 frames or rows t [F, ...] (a view into a Guarded buffer): randn (|randn| with relu), odd ones and F-2 relu(randn) + 3 (mean /
    spread ~ 6), the last one 3 + randn * 3/64; generated in chunks"""
    Fn = t.shape[0]
    per = t[0].numel()
    g = torch.Generator(device=DEV).manual_seed(seed)
    step = max(1, (1 << 26) // per)
    for f0 in range(0, Fn, step):
        f1 = min(Fn, f0 + step)
        x = torch.randn((f1 - f0,) + tuple(t.shape[1:]), generator=g, device=DEV)
        if relu:
            x = x.abs()
        for f in range(f0, f1):
            k = frame_kind(f, Fn)
            if k == "dc":
                x[f - f0] = x[f - f0].relu() + 3.0
            elif k == "const":
                x[f - f0] = 3.0 + x[f - f0] * (3.0 / 64)
        t[f0:f1] = x
    return t


def frames(Fn, H, W, seed, dtype):
    """[F, H, W, 3] pixels on the uint8 scale, uint8 or non-integer fp32: uniform; odd frames and F-2 180 + 30 randn (mean / spread 6);
    the last frame 128 + 2 randn"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand((Fn, H, W, 3), generator=g, device=DEV) * 255
    for f in range(Fn):
        k = frame_kind(f, Fn)
        if k != "randn":
            m, s = (180.0, 30.0) if k == "dc" else (128.0, 2.0)
            x[f] = m + s * torch.randn((H, W, 3), generator=g, device=DEV)
    x = x.clamp(0, 255)
    return x.round().to(U8) if dtype == U8 else x


def guarded(shape, dtype=F32):
    n = 1
    for s in shape:
        n *= s
    b = Guarded(n, dtype)
    return b, b.t.view(*shape)


def check(name, out, ref, kinds, l2_bound, max_bound):
    """per checked row / frame: rel-L2 and max |err| / rms(ref); the worst of each kind against the bounds"""
    o = out.reshape(out.shape[0], -1).to(F64)
    r = ref.reshape(ref.shape[0], -1)
    d = o - r
    rms = r.pow(2).mean(1).sqrt().clamp(min=1e-300)
    l2 = d.norm(dim=1) / (rms * r.shape[1] ** 0.5)
    mx = d.abs().amax(1) / rms
    ok = bool(torch.isfinite(o).all())
    for k in dict.fromkeys(kinds):
        j = [i for i, kk in enumerate(kinds) if kk == k]
        e2, em = l2[j].max().item(), mx[j].max().item()
        print(f"{name} [{k}]: rel-L2 {e2:.2e} (bound {l2_bound:.0e}), max |err| / rms {em:.2e} (bound {max_bound:.0e})")
        ok = ok and e2 <= l2_bound and em <= max_bound
    assert ok, name


def check_stats(name, mr, x, kinds):
    """group_stats_f32's (mean, rstd) [G][2] against float64 of its input x [G, ...]"""
    ref = Rf.stats(x)
    e_m = (mr[:, 0].to(F64) - ref[:, 0]).abs() * ref[:, 1]
    e_r = (mr[:, 1].to(F64) - ref[:, 1]).abs() / ref[:, 1]
    for k in dict.fromkeys(kinds):
        j = [i for i, kk in enumerate(kinds) if kk == k]
        print(f"{name} [{k}]: |d mean| * rstd {e_m[j].max().item():.2e} (bound {STAT_MEAN:.0e}), |d rstd| / rstd {e_r[j].max().item():.2e} "
              f"(bound {STAT_RSTD:.0e})")
    assert torch.isfinite(mr).all() and e_m.max().item() <= STAT_MEAN and e_r.max().item() <= STAT_RSTD, name


def snap(t):
    """what _run_twice compares: the tensor itself, or its per-row digest when large"""
    return digest(t) if t.numel() > (1 << 24) else t.clone()


def norm_gemm(name, xb, x, groups, norm, Wsplit, M, N, K, *, conv=None, bias=None, relu=False, out_scale=1.0, ld=None):
    """precise._norm_gemm (norm = (gamma, beta) with groups, or the plain split of `norm_split_f32(x)` with norm = None) into guarded
    buffers: vpt_group_stats_f32 -> vpt_norm_split_f32 -> precise.gemm3.  Returns (out [M][ld], mr or None) after two bit-identical calls."""
    n = x.numel()
    C = x.shape[-1]
    ld = ld or N
    mb = Guarded(groups * 2) if norm is not None else None
    hb, lb = Guarded(n, BF16), Guarded(n, BF16)
    ab, ob = Guarded(M * ld), Guarded(M * ld)
    acc, out = ab.t.view(M, ld), ob.t.view(M, ld)
    mr = mb.t.view(groups, 2) if mb is not None else None
    gamma, beta = norm if norm is not None else (None, None)
    bufs = [b for b in (xb, mb, hb, lb, ab, ob) if b is not None]

    def call():
        refill(*bufs[1:])
        if mr is not None:
            nat.check(lib().vpt_group_stats_f32(x.data_ptr(), mr.data_ptr(), groups, n // groups, 1e-5, stream()), "vpt_group_stats_f32")
        nat.check(lib().vpt_norm_split_f32(x.data_ptr(), _p(mr), _p(gamma), _p(beta), hb.ptr(), lb.ptr(), None, n, C, n // groups if mr is not None else 0,
                                           stream()), "vpt_norm_split_f32")
        P.gemm3(hb.t.view(M, K) if conv is None else hb.t, lb.t.view(M, K) if conv is None else lb.t, Wsplit, M, N, K, conv=conv, bias=bias,
                relu=relu, out_scale=out_scale, ld=ld, acc=acc, out=out)
        return [snap(out[:, :N]), snap(acc[:, :N])] + ([mr.clone()] if mr is not None else []), bufs

    _run_twice(name, call)
    assert all_finite(out[:, :N]) and all_finite(acc[:, :N]) and all_finite(hb.t[None]) and all_finite(lb.t[None]), name
    del hb, lb, ab, acc
    return ob, out, mr


# ---------------------------------------------------------------------------------------------------------------------
# the CNN
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Fn", [1, 3, 512])
def test_stack0_firstconv_pool_f32(model, Fn):
    """stack 0 of the agents: vpt_firstconv_pool(_f32) with zp = 0, out_f32 = 1 (blocks of 64 channels: C0 = 192 takes three) on uint8 and
    on non-integer fp32 frames, against float64 fanin_conv -> max_pool2d"""
    w, s, pol, sd, prep = model
    if s["firstconv"] is None:
        pytest.skip("the IDM's stack 0 opens with the conv3d pre-stage and a normalised conv (test_normalised_convs)")
    st, C0 = prep.stacks[0], s["firstconv"]
    H, W = s["stacks"][0]["H"], s["stacks"][0]["W"]
    idx = sel_frames(Fn)
    kinds = [frame_kind(f, Fn) for f in idx]
    for dt in (U8, F32):
        ib, img = guarded((Fn, H, W, 3), dt)
        img.copy_(frames(Fn, H, W, Fn, dt))
        Pn = lib().vpt_firstconv_stat_parts(Fn, H, W, C0)
        ob, out = guarded((Fn, H // 2, W // 2, C0))
        pb = Guarded(Fn * Pn * 2)
        fn = "vpt_firstconv_pool_f32" if dt == F32 else "vpt_firstconv_pool"
        name = f"{w} {fn} out_f32 C0={C0} F={Fn}"

        def call():
            refill(ob, pb)
            nat.check(getattr(lib(), fn)(img.data_ptr(), st["fc_w"].data_ptr(), st["fc_b"].data_ptr(), out.data_ptr(), pb.ptr(), Fn, H, W, C0, 0, 1,
                                         stream()), fn)
            return [snap(out), pb.t.clone()], [ib, ob, pb]

        _run_twice(name, call)
        assert all_finite(out) and all_finite(pb.t[None])
        check(name, out[idx], Rf.firstconv_pool(img[idx], sd, "img_process.cnn.stacks.0"), kinds, FC_L2, FC_MAX)
        del ib, img, ob, out, pb


@pytest.mark.parametrize("B", [1, 4])
def test_idm_conv3d_pre_stage_f32(model, B):
    """vpt_conv3d_t5(_f32) with out_f32 = 1 at B x 128 frames on uint8 and fp32 frames: the ZP pad row and column come back 0, the
    interior against float64 conv3d_stage on the frames at both ends of every sequence and one between"""
    w, s, pol, sd, prep = model
    if s["conv3d"] is None:
        pytest.skip("the policies have no conv3d pre-stage")
    H, W, _ = s["cfg"].img_shape
    Cc, T = s["conv3d"], s["t"]
    w3, b3 = prep.conv3d
    Fn = B * T
    for dt in (U8, F32):
        ib, img = guarded((B, T, H, W, 3), dt)
        img.view(Fn, H, W, 3).copy_(frames(Fn, H, W, 40 + B, dt))
        Pn = lib().vpt_conv3d_stat_parts(H, W, Cc)
        ob, out = guarded((Fn, H + 1, W + 1, Cc))
        pb = Guarded(Fn * Pn * 2)
        fn = "vpt_conv3d_t5_f32" if dt == F32 else "vpt_conv3d_t5"
        name = f"{w} {fn} out_f32 B={B} T={T}"

        def call():
            refill(ob, pb)
            nat.check(getattr(lib(), fn)(img.data_ptr(), w3.data_ptr(), b3.data_ptr(), out.data_ptr(), pb.ptr(), B, T, H, W, Cc, 1, stream()), fn)
            return [snap(out), pb.t.clone()], [ib, ob, pb]

        _run_twice(name, call)
        assert all_finite(out) and all_finite(pb.t[None])
        assert bool((out[:, -1] == 0).all()) and bool((out[:, :, -1] == 0).all()), f"{name}: the ZP pad row / column is not 0"
        ref, fr = [], []
        for b in range(B):
            for t in (0, 1, T // 2, T - 2, T - 1):
                lo, hi = max(0, t - 2), min(T, t + 3)
                ref.append(Rf.conv3d(img[b:b + 1, lo:hi], sd, "conv3d_layer")[t - lo])
                fr.append(b * T + t)
        kinds = [frame_kind(f, Fn) for f in fr]
        check(name, out[fr][:, :-1, :-1], torch.stack(ref), kinds, FC_L2, FC_MAX)
        del ib, img, ob, out, pb


def _conv_stage(w, s, sd, prep, i, Fn, first):
    """one normalised conv of stack i (first: the stack's first conv at its input size, else the four block convs at the pooled size)"""
    sh = s["stacks"][i]
    p = f"img_process.cnn.stacks.{i}"
    st = prep.stacks[i]
    if first:
        H, W, Cin, Cc = sh["H"], sh["W"], sh["Cin"], sh["C"]
        convs = [(p + ".firstconv", st["first"])]
    else:
        H, W, Cin, Cc = sh["H"] // 2, sh["W"] // 2, sh["C"], sh["C"]
        convs = [(f"{p}.blocks.{j}.conv{k}", st["convs"][2 * j + k]) for j in range(2) for k in range(2)]
    idx = sel_frames(Fn)
    kinds = [frame_kind(f, Fn) for f in idx]
    for c, (pre, (Wsplit, gam, bet)) in enumerate(convs):
        xb, x = guarded((Fn, H, W, Cin))
        fill32(x, 100 * i + 10 * c + Fn, relu=c % 2 == 1)  # the second conv of a block reads the first one's ReLU output
        name = f"{w} stack {i} {pre.split('.', 4)[-1]} {H}x{W} {Cin}->{Cc} F={Fn}"
        ob, out, mr = norm_gemm(name, xb, x, Fn, (gam, bet), Wsplit, Fn * H * W, Cc, 9 * Cin, conv=(H, W, Cin), relu=True)
        check_stats(f"{name} (mean, rstd)", mr[idx], x[idx], kinds)
        check(name, out.view(Fn, H, W, Cc)[idx], Rf.conv_nhwc(x[idx], sd, pre), kinds, CONV_L2, CONV_MAX)
        del xb, x, ob, out, mr


@pytest.mark.parametrize("Fn", [1, 3, 128])
def test_normalised_convs(model, Fn):
    """every normalised conv -- each stack's first conv (the IDM's stack 0 included) and its four block convs -- as precise._norm_gemm
    runs it: group_stats_f32 -> norm_split_f32 -> gemm3 (plain-NHWC implicit GEMM) -> ReLU, against float64 fanin_conv"""
    w, s, pol, sd, prep = model
    for i, sh in enumerate(s["stacks"]):
        if not sh["fused_first"]:
            _conv_stage(w, s, sd, prep, i, Fn, first=True)
        _conv_stage(w, s, sd, prep, i, Fn, first=False)


@pytest.mark.parametrize("Fn", [1, 3, 128])
def test_pool_norm_and_residual(model, Fn):
    """per stack: vpt_maxpool3s2_f32 (bit-exact with float64 max_pool2d), the post-pool GroupNorm as precise.forward runs it
    (group_stats_f32 -> norm_split_f32 without the split, fp32 out) against float64 F.group_norm, and vpt_add_f32 (bit-exact with the fp32
    sum, with and without ReLU)"""
    w, s, pol, sd, prep = model
    idx = sel_frames(Fn)
    kinds = [frame_kind(f, Fn) for f in idx]
    for i, sh in enumerate(s["stacks"]):
        H, W, Cc = sh["H"], sh["W"], sh["C"]
        Ho, Wo = H // 2, W // 2
        name = f"{w} stack {i} maxpool3s2_f32 {H}x{W}x{Cc} F={Fn}"
        xb, x = guarded((Fn, H, W, Cc))
        fill32(x, 500 + i, relu=True)
        yb, y = guarded((Fn, Ho, Wo, Cc))

        def pool():
            refill(yb)
            nat.check(lib().vpt_maxpool3s2_f32(x.data_ptr(), y.data_ptr(), Fn, H, W, Cc, stream()), "vpt_maxpool3s2_f32")
            return [snap(y)], [xb, yb]

        _run_twice(name, pool)
        assert all_finite(y)
        bad = (y[idx].to(F64) != Rf.maxpool_nhwc(x[idx])).sum().item()
        print(f"{name}: mismatches against float64 max_pool2d {bad} (bound 0)")
        assert bad == 0, name
        del xb, x
        n = y.numel()
        mb, nb = Guarded(Fn * 2), Guarded(n)
        mr, u = mb.t.view(Fn, 2), nb.t.view(y.shape)
        st = prep.stacks[i]
        name = f"{w} stack {i} post-pool GroupNorm {Ho}x{Wo}x{Cc} F={Fn}"

        def norm():
            refill(mb, nb)
            nat.check(lib().vpt_group_stats_f32(y.data_ptr(), mr.data_ptr(), Fn, n // Fn, 1e-5, stream()), "vpt_group_stats_f32")
            nat.check(lib().vpt_norm_split_f32(y.data_ptr(), mr.data_ptr(), st["n"][0].data_ptr(), st["n"][1].data_ptr(), None, None, u.data_ptr(), n,
                                               Cc, n // Fn, stream()), "vpt_norm_split_f32")
            return [mr.clone(), snap(u)], [yb, mb, nb]

        _run_twice(name, norm)
        assert all_finite(u) and all_finite(mr)
        check_stats(f"{name} (mean, rstd)", mr[idx], y[idx], kinds)
        check(name, u[idx], Rf.group_norm_nhwc(y[idx], sd, f"img_process.cnn.stacks.{i}.n"), kinds, NORM_L2, NORM_MAX)
        del yb, y, mb, mr
        rb, r = guarded(u.shape)
        fill32(r, 600 + i)
        sb, sm = guarded(u.shape)
        for relu in (0, 1):
            def add():
                refill(sb)
                nat.check(lib().vpt_add_f32(u.data_ptr(), r.data_ptr(), sm.data_ptr(), n, relu, stream()), "vpt_add_f32")
                return [snap(sm)], [nb, rb, sb]

            _run_twice(f"{w} stack {i} add_f32 relu={relu} F={Fn}", add)
            ref = u[idx] + r[idx]
            bad = (sm[idx] != (ref.relu() if relu else ref)).sum().item()
            print(f"{w} stack {i} add_f32 relu={relu} F={Fn}: mismatches against the fp32 sum {bad} (bound 0)")
            assert all_finite(sm) and bad == 0
        del nb, u, rb, r, sb, sm


# ---------------------------------------------------------------------------------------------------------------------
# linear layers, heads
# ---------------------------------------------------------------------------------------------------------------------
def _rows(M, K, seed, relu=False):
    b, x = guarded((M, K))
    fill32(x, seed, relu=relu)
    return b, x


def _linear(name, x, xb, M, idx, ref, *, norm=None, W, N, K, bias=None, relu=False, out_scale=1.0, ld=None):
    kinds = [frame_kind(r, M) for r in idx]
    tc = M > 8  # the small-M kernel below
    l2, mx = (VALUE_REL, VALUE_REL) if N == 1 else (LIN_L2 + tc * TC_L2_PER_K * K, LIN_MAX + tc * TC_MAX_PER_K * K)
    ob, out, mr = norm_gemm(name, xb, x, M, norm, W, M, N, K, bias=bias, relu=relu, out_scale=out_scale, ld=ld)
    if mr is not None:
        check_stats(f"{name} (mean, rstd)", mr[idx], x[idx], kinds)
    check(name, out[idx, :N], ref, kinds, l2, mx)
    return ob, out


@pytest.mark.parametrize("M", [1, 8, 9, 200, 2048])
def test_linear_layers(model, M):
    """dense (K = 32 768 .. 131 072, rows flattened H, W, C), linear, q / k / v / R (the LayerNorm of the block, R's ld), proj, mlp0,
    mlp1 (+ add_f32, with ReLU after the last block), lastlayer, as precise.forward calls them; M <= 8 runs on the small-M kernel, 9 is the
    smallest M on the tensor cores"""
    w, s, pol, sd, prep = model
    cfg = s["cfg"]
    Hf, Wf, C2, _ = s["dense"]
    h, heads = s["h"], s["heads"]
    idx = sel_frames(M)
    L = len(prep.layers) - 1
    Lp = prep.layers[L]
    b = f"recurrent_layer.blocks.{L}"
    o = b + ".r.orc_block"
    Kd = Hf * Wf * C2
    xb, x = _rows(M, Kd, 1)
    Wd, gd, bd = prep.dense
    ref = Rf.linear(Rf.dense_from_nhwc(x[idx], Hf, Wf, C2), sd, "img_process.cnn.dense")
    _linear(f"{w} dense {Kd}->{cfg.cnn_outsize} M={M}", x, xb, M, idx, ref, norm=(gd, bd), W=Wd, N=cfg.cnn_outsize, K=Kd, relu=True)
    del xb, x
    xb, x = _rows(M, cfg.cnn_outsize, 2)
    Wl, gl, bl = prep.linear
    _linear(f"{w} linear M={M}", x, xb, M, idx, Rf.linear(x[idx], sd, "img_process.linear"), norm=(gl, bl), W=Wl, N=h, K=cfg.cnn_outsize, relu=True)
    # the attention block's projections read the split of LayerNorm(x) (norm_split_f32 with the block's pre_r_ln)
    xb, x = _rows(M, h, 3)
    xn = Rf.layer_norm(x[idx], sd, b + ".pre_r_ln")
    R_ld = (10 * heads + 3) // 4 * 4
    for nm, (Wq, bq), N, ld in [("q", Lp["q"], h, None), ("k", Lp["k"], h, None), ("v", Lp["v"], h, None)] + \
            ([("R", Lp["r"], 10 * heads, R_ld)] if s["causal"] else []):
        lay = {"q": "q_layer", "k": "k_layer", "v": "v_layer", "R": "r_layer"}[nm]
        ref = Rf.plain_linear(xn, sd, f"{o}.{lay}", bias=bq is not None)
        _linear(f"{w} {nm} {h}->{N} ld={ld or N} M={M}", x, xb, M, idx, ref, norm=Lp["ln"], W=Wq, N=N, K=h, bias=bq, ld=ld)
    y = x  # the residual stream
    ab, a = _rows(M, h, 4)
    ob, pr = _linear(f"{w} proj M={M}", a, ab, M, idx, Rf.plain_linear(a[idx], sd, o + ".proj_layer"), W=Lp["proj"][0], N=h, K=h, bias=Lp["proj"][1])
    del ab, a
    _add(f"{w} proj + x_hat M={M}", y, pr, 0, [xb, ob])
    del ob, pr
    W0, g0, b0 = Lp["mlp0"]
    _linear(f"{w} mlp0 M={M}", y, xb, M, idx, Rf.linear(y[idx], sd, b + ".mlp0"), norm=(g0, b0), W=W0, N=h * cfg.pointwise_ratio, K=h, relu=True)
    hb, hm = _rows(M, h * cfg.pointwise_ratio, 5, relu=True)
    ref = Rf.linear(hm[idx], sd, b + ".mlp1", relu=False)
    ob, m1 = _linear(f"{w} mlp1 M={M}", hm, hb, M, idx, ref, W=Lp["mlp1"][0], N=h, K=h * cfg.pointwise_ratio, bias=Lp["mlp1"][1])
    del hb, hm
    for relu in (0, 1):
        _add(f"{w} mlp1 + y relu={relu} M={M}", y, m1, relu, [xb, ob])
    del ob, m1
    if "lastlayer" in s["linears"]:
        zb, z = _rows(M, h, 6, relu=True)
        Wt, gt, bt = prep.last
        _linear(f"{w} lastlayer M={M}", z, zb, M, idx, Rf.linear(z[idx], sd, "lastlayer"), norm=(gt, bt), W=Wt, N=h, K=h, relu=True)


def _add(name, a, b, relu, in_bufs):
    M, N = a.shape
    sb, out = guarded((M, N))

    def call():
        refill(sb)
        nat.check(lib().vpt_add_f32(a.data_ptr(), b.data_ptr(), out.data_ptr(), M * N, relu, stream()), "vpt_add_f32")
        return [out.clone()], in_bufs + [sb]

    _run_twice(name, call)
    ref = a + b[:, :N]
    bad = (out != (ref.relu() if relu else ref)).sum().item()
    print(f"{name}: mismatches against the fp32 sum {bad} (bound 0)")
    assert bad == 0, name


@pytest.mark.parametrize("M", [1, 8, 9, 200, 2048])
def test_heads(model, M):
    """the action heads as precise.heads runs them: gemm3 with bias, out_scale = 1 / temperature and N = ntot written into ld = ntot rounded
    up to 8; the value head (N = 1, ld = 4); against float64 F.linear of the fp32 latent"""
    w, s, pol, sd, prep = model
    hp = pol._heads_prepared_precise()
    N, ld, h, temp = s["ntot"], s["ld_logits"], s["h"], pol.temperature
    assert hp["ntot"] == N and (N + 7) // 8 * 8 == ld
    idx = sel_frames(M)
    lb, lat = _rows(M, h, 7)
    Wt = torch.cat([getattr(pol.pi_head, name).linear_layer.weight for name, *_ in s["head_cols"]]).to(F64)
    bias = torch.cat([getattr(pol.pi_head, name).linear_layer.bias for name, *_ in s["head_cols"]]).to(F64)
    ref = F.linear(lat[idx].to(F64), Wt, bias) / temp
    _linear(f"{w} pi head N={N} ld={ld} 1/T={1 / temp:g} M={M}", lat, lb, M, idx, ref, W=hp["pi"][0], N=N, K=h, bias=hp["pi"][1],
            out_scale=1.0 / temp, ld=ld)
    if pol.has_value_head:
        lin = pol.value_head.linear
        ref = F.linear(lat[idx].to(F64), lin.weight.to(F64), lin.bias.to(F64))
        _linear(f"{w} value head N=1 ld=4 M={M}", lat, lb, M, idx, ref, W=hp["v"][0], N=1, K=h, bias=hp["v"][1], ld=4)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def _attention(name, B, t, maxlen, heads, causal, seed, b_nd=None):
    """vpt_attention_f32 on guarded fp32 inputs (causal: a state mask with holes, `first` set on rows 1, 4, 7, ...) against float64"""
    h = heads * 128
    T = maxlen + t
    g = torch.Generator(device=DEV).manual_seed(seed)
    bufs = dict(Q=guarded((B * t, h)), Kf=guarded((B, T, h)), Vf=guarded((B, T, h)))
    if causal:
        bufs.update(R=guarded((B * t, 10 * heads)), b_nd=guarded((10, maxlen)), first_u8=guarded((B, t), U8), smask_u8=guarded((B, maxlen), U8))
    x = {k: v[1] for k, v in bufs.items()}
    x["Q"].copy_(torch.randn(x["Q"].shape, generator=g, device=DEV) * 3)
    x["Kf"].copy_(torch.randn(x["Kf"].shape, generator=g, device=DEV) * 3)
    x["Vf"].copy_(torch.randn(x["Vf"].shape, generator=g, device=DEV))
    if causal:
        x["R"].copy_(torch.randn(x["R"].shape, generator=g, device=DEV))
        x["b_nd"].copy_(b_nd if b_nd is not None else torch.randn((10, maxlen), generator=g, device=DEV) * 0.5)
        x["first_u8"].zero_()
        x["first_u8"][1::3, 0] = 1
        x["smask_u8"].copy_((torch.rand((B, maxlen), generator=g, device=DEV) > 0.3).to(U8))
    ob, out = guarded((B * t, h))

    def call():
        refill(ob)
        nat.check(lib().vpt_attention_f32(x["Q"].data_ptr(), x["Kf"].data_ptr(), x["Vf"].data_ptr(), _p(x.get("R")), _p(x.get("b_nd")),
                                          _p(x.get("first_u8")), _p(x.get("smask_u8")), out.data_ptr(), B, t, maxlen, heads, int(causal), stream()),
                  "vpt_attention_f32")
        return [out.clone()], [v[0] for v in bufs.values()] + [ob]

    _run_twice(name, call)
    assert all_finite(out)
    if causal:
        ref = attention_ref(x, B, t, maxlen, heads)
    else:
        q = x["Q"].to(F64).reshape(B, t, heads, 128).transpose(1, 2)
        k = x["Kf"].to(F64).reshape(B, T, heads, 128).transpose(1, 2)
        v = x["Vf"].to(F64).reshape(B, T, heads, 128).transpose(1, 2)
        ref = (torch.softmax(q @ k.transpose(-1, -2) / 128, -1) @ v).transpose(1, 2).reshape(B * t, h)
    # per query and head: every query of every (batch row, head) pair, as rows of 128
    got, want = out.view(B * t * heads, 128), ref.view(B * t * heads, 128)
    fst = x["first_u8"][:, 0].tolist() if causal else [0] * B
    kinds = ["first" if fst[r // (t * heads)] else "memory" if causal else "unmasked" for r in range(B * t * heads)]
    check(name, got, want, kinds, ATTN_L2, ATTN_MAX)


@pytest.mark.parametrize("t,B", [(128, 4), (1, 64)])
def test_attention_at_the_model_heads(model, t, B):
    """vpt_attention_f32 at the model's heads and maxlen 128 with its own b_nd (the IDM: unmasked, t = 128, B = 4)"""
    w, s, pol, sd, prep = model
    heads, maxlen = s["heads"], s["maxlen"]
    if not s["causal"]:
        if t != 128:
            pytest.skip("the IDM runs whole 128-frame chunks")
        _attention(f"{w} attention_f32 unmasked heads={heads} t={t} B={B}", B, t, maxlen, heads, False, 20)
        return
    _attention(f"{w} attention_f32 heads={heads} t={t} maxlen={maxlen} B={B}", B, t, maxlen, heads, True, 21 + t,
               b_nd=prep.layers[0]["b_nd"])


@pytest.mark.parametrize("B,t,maxlen,heads", [(2, 128, 1920, 16), (1, 1, 12287, 1), (1, 1, 16000, 1)])
def test_attention_long_memory(B, t, maxlen, heads):
    """long KV memories: the reference's default (maxlen 1920) at t = 128; exactly 12 288 keys, whose 48 KB score row with the kernel's
    static shared memory needs the opt-in above the default limit; and 16 001 keys"""
    _attention(f"attention_f32 heads={heads} t={t} maxlen={maxlen} B={B}", B, t, maxlen, heads, True, maxlen + t)


def test_attention_rejects_more_than_51200_keys():
    """argument validation: the score row of more than 51 200 keys does not fit the 200 KB of shared memory; nothing is launched"""
    z = torch.zeros(128, device=DEV)
    u = torch.zeros(1, dtype=U8, device=DEV)
    with pytest.raises(nat.NativeError, match="keys"):
        nat.check(lib().vpt_attention_f32(z.data_ptr(), z.data_ptr(), z.data_ptr(), None, None, u.data_ptr(), u.data_ptr(), z.data_ptr(), 1, 1, 51200, 1, 1,
                                          stream()), "vpt_attention_f32")
    nat.device_check()
