"""Backward kernels of the training steps at the shapes they reach (B x T = 2048 frames / tokens at the widths 1x / 2x / 3x, 512 for the
4x IDM), against the float64 references of tests/bwd_refs.py, plus: every write stays inside its declared buffer, every reduction is
bit-reproducible, and the whole 3x-width step matches forced autograd.

The conv side runs F = 16..128 frames instead of 2048: F is the smallest count whose launch plan (wgrad K splits, norm slabs) equals
the production one, read back from the library's own workspace queries.  Each check prints its measured error beside its bound."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import bwd_refs as Rf
import vpt_b200
from common import make_policy
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import _rot
from video_pre_training_b200.training import BCTrainer

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
WIDTHS = ["1x", "2x", "3x"]
MODELS = WIDTHS + ["idm"]  # the IDM where a test body takes its shapes unchanged
SHAPES = {w: Rf.backward_shapes(w) for w in MODELS}
ROWS = SHAPES["3x"]["N"]  # tokens of a training step (B = 16, T = 128)

# Bounds: each is at most 4x the worst value measured on an H100 80GB HBM3 (SXM) at a 400 W power limit, given beside it.
# Weight gradients: the fp32 accumulation error grows with the rows one CTA sums (R / splits), so the bounds are per summed row:
# measured 3.9e-10 (|err| / sum|a||b|) and 1.06e-9 (rel-L2) per row, conv and linear alike.
WG_ELEM_ROW, WG_L2_ROW = 1.5e-9, 4e-9
BF_FLOOR_CONV = 8e-6            # dgrad conv: |err| <= 2^-8 |ref| + floor * (max |ref| of the pixel); measured 2.1e-6
BF_FLOOR_NORM = 1.2e-9          # norm dx; measured 2.9e-10
# norm dx + add with relu_x: where dx and add nearly cancel the fp32 error of dx shows above 2^-8 |ref|; measured 3.6e-8 (H100 80GB HBM3,
# 700 W)
BF_FLOOR_NORM_ADD = 1.4e-7
BF_FLOOR_ATTN = 6e-7            # dq / dk / dv / dR; measured 1.6e-7
BF_FLOOR_SOFTMAX = 0.0          # measured < 0: every element within 2^-8 |ref|
BF_FLOOR_GROUPED = 2.3e-7       # the IDM's grouped heads: exp(logp) - 1 near p = 1 cancels; measured 5.7e-8 (H100 80GB HBM3, 700 W)
NORM_ELEM, NORM_L2 = 3e-7, 6e-7  # ms, dgamma, dbeta: |err| / (sum of the absolute terms), rel-L2; measured 7.6e-8, 1.4e-7
FC_L2 = 4e-7                    # first conv dW / db rel-L2; measured 9.5e-8
DBND_L2 = 1.1e-6                # attention d b_nd rel-L2; measured 2.7e-7
DLOG_ELEM, DLOG_L2 = 1.3e-6, 2.4e-7  # head bias sums over 2048 rows; measured 3.3e-7, 6.0e-8


def lib():
    return nat.lib()


def stream():
    return torch.cuda.current_stream().cuda_stream


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=g, device=DEV) * scale + shift


def zp(x_nhwc):
    """[F,H,W,C] -> bf16 ZP [F,H+1,W+1,C] with zero pads"""
    return F.pad(x_nhwc.to(BF16), (0, 0, 0, 1, 0, 1))


def rel(a, b):
    return ((a.to(F64) - b.to(F64)).norm() / b.to(F64).norm()).item()


def check_sum(name, out, ref, scale, elem, l2):
    """fp32 result of a sum against the float64 sum; `scale` = the same sum over absolute values"""
    e = ((out.to(F64) - ref).abs() / scale.clamp(min=1e-300)).max().item()
    r = rel(out, ref)
    print(f"{name}: max |err|/sum|terms| {e:.2e} (bound {elem:.0e}), rel-L2 {r:.2e} (bound {l2:.0e})")
    assert e <= elem and r <= l2, name


def check_bf16(name, out, ref, floor):
    """bf16 result: |out - ref| <= 2^-8 |ref| + floor * (max |ref| over the last dimension)"""
    d = (out.to(F64) - ref).abs()
    rowmax = ref.abs().amax(-1, keepdim=True).clamp(min=1e-300)
    excess = ((d - 2 ** -8 * ref.abs()) / rowmax).max().item()
    print(f"{name}: rel-L2 {rel(out, ref):.2e}, max (|err| - 2^-8 |ref|) / row max {excess:.2e} (bound {floor:.0e})")
    assert torch.isfinite(out).all() and excess <= floor, name


def wgrad_splits(M, N, ntaps, R):
    return max(1, lib().vpt_wgrad_workspace_bytes(M, N, ntaps, R) // (4 * M * N * ntaps))


def wgrad_bounds(M, N, ntaps, R):
    rows = R / wgrad_splits(M, N, ntaps, R)
    return WG_ELEM_ROW * rows, WG_L2_ROW * rows


def conv_shifts(W):
    return [(ky - 1) * (W + 1) + (kx - 1) for ky in range(3) for kx in range(3)]


def frames_for_plan(plan, per_frame, lo=16, hi=128, rows=ROWS):
    """smallest frame count in [lo, hi] (steps of 8) whose launch plan equals the one at `rows` frames"""
    want = plan(rows * per_frame)
    for Fn in range(lo, hi + 1, 8):
        if plan(Fn * per_frame) == want:
            return Fn, want
    pytest.fail(f"no frame count <= {hi} reproduces the production plan {want}")


# ---------------------------------------------------------------------------------------------------------------------
# weight gradients and dgrad convolutions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", MODELS)
def test_conv_wgrad_and_dgrad_at_production_plans(width):
    for i, (H, W, Cin, Cout) in enumerate(SHAPES[width]["convs"]):
        P = (H + 1) * (W + 1)
        Fn, splits = frames_for_plan(lambda R: wgrad_splits(Cout, Cin, 9, R), P, rows=SHAPES[width]["N"])
        if Cout <= 128:  # one (M, N) tile: the production plan splits K over > 16 CTAs (30 on 132 SMs)
            assert splits > 16, (H, W, Cin, Cout, splits)
        g = gen(10 + i)
        dz = zp(randn((Fn, H, W, Cout), g).relu())          # the ReLU-masked output gradient
        u = zp(randn((Fn, H, W, Cin), g, 0.8, 0.2))        # the normalised layer input
        dW = ops.wgrad(dz.view(-1, Cout), u.view(-1, Cin), conv_shifts(W))
        ref, scale = Rf.conv_wgrad(dz, u)
        check_sum(f"{width} wgrad conv {H}x{W} {Cin}->{Cout} F={Fn} splits={splits}", dW, ref, scale, *wgrad_bounds(Cout, Cin, 9, dz.shape[0] * P))
        Wt = randn((Cout, Cin, 3, 3), g, (2.0 / (9 * Cin)) ** 0.5).to(BF16)
        du, _ = ops.conv3x3_zp(dz, _rot(Wt), H, W, relu=0, want_stats=False)
        ref, _ = Rf.conv_dgrad(dz, Wt)
        assert (du[:, -1] == 0).all() and (du[:, :, -1] == 0).all()
        check_bf16(f"{width} dgrad conv {H}x{W} {Cout}->{Cin} F={Fn}", du, ref, BF_FLOOR_CONV)
    nat.device_check()


def test_wgrad_at_the_split_cap_with_a_ragged_last_split():
    """637 K iterations of 64 rows: 64 splits of 10, the last one 7 iterations long, ending in a 44-row K tail."""
    M = N = 128
    R = 636 * 64 + 44
    assert wgrad_splits(M, N, 1, R) == 64
    g = gen(20)
    a, b = randn((R, M), g).to(BF16), randn((R, N), g).to(BF16)
    ref, scale = Rf.linear_wgrad(a, b)
    check_sum("wgrad split cap", ops.wgrad(a, b), ref, scale, *wgrad_bounds(M, N, 1, R))
    nat.device_check()


@pytest.mark.parametrize("width", MODELS)
def test_linear_wgrad_at_production_shapes(width):
    rows = SHAPES[width]["N"]
    for i, (M, N) in enumerate(SHAPES[width]["linears"]):
        g = gen(30 + i)
        a, b = randn((rows, M), g).to(BF16), randn((rows, N), g).to(BF16)
        ref, scale = Rf.linear_wgrad(a, b)
        check_sum(f"{width} wgrad linear {M}x{N} rows={rows} splits={wgrad_splits(M, N, 1, rows)}", ops.wgrad(a, b), ref, scale,
                  *wgrad_bounds(M, N, 1, rows))
        del ref, scale
    nat.device_check()


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm / LayerNorm backward
# ---------------------------------------------------------------------------------------------------------------------
def _norm_case(name, G, rpg, C, zpg, seed, fused=False):
    """fused: x is a ReLU output (about a third zeros) and the apply pass also takes `add` and `relu_x`, as for a norm whose input feeds a
    residual too (add) or comes out of a ReLU (relu_x)"""
    g = gen(seed)
    act = (lambda v: v.relu()) if fused else (lambda v: v)
    if zpg is not None:
        H, W, Cc = zpg
        x = zp(act(randn((G, H, W, Cc), g, 0.7, 0.3))).reshape(G * rpg, C)
        du = zp(randn((G, H, W, Cc), g)).reshape(G * rpg, C)
        add = zp(randn((G, H, W, Cc), g)).reshape(G * rpg, C) if fused else None
        count = H * W * Cc
    else:
        x, du = act(randn((G, C), g, 0.7, 0.3)).to(BF16), randn((G, C), g).to(BF16)
        add = randn((G, C), g).to(BF16) if fused else None
        count = C
    gamma = randn((C,), g, 0.3, 1.0)
    mr = Rf.norm_stats(x, rpg, zpg)
    ref = Rf.norm_bwd(du, x, gamma, rpg, zpg, add=add, relu_x=fused)
    if rpg > 1:
        cs, ms = ops.norm_sums(du, x, mr, gamma, rpg, count)
    else:
        cs, ms = ops.col_sums(du, x, mr, rpg), ops.group_sums(du, x, mr, gamma, rpg, count)
    grp = torch.arange(x.shape[0], device=DEV) // rpg
    n = (x.to(F64) - mr[grp, 0:1].to(F64)) * mr[grp, 1:2].to(F64)
    gdu = (du.to(F64) * gamma.to(F64)).abs()
    ms_scale = torch.stack([gdu.reshape(-1, rpg * C).sum(1), (gdu * n.abs()).reshape(-1, rpg * C).sum(1)], 1) / count
    check_sum(f"{name} ms", ms, ref["ms"], ms_scale, NORM_ELEM, NORM_L2)
    check_sum(f"{name} dgamma", cs[0], ref["dgamma"], (du.to(F64).abs() * n.abs()).sum(0), NORM_ELEM, NORM_L2)
    check_sum(f"{name} dbeta", cs[1], ref["dbeta"], du.to(F64).abs().sum(0), NORM_ELEM, NORM_L2)
    dx = ops.norm_bwd_apply(du, x, mr, gamma, ref["ms"].float(), rpg, zp=zpg, add=add, relu_x=fused)
    if fused:
        name = f"{name} (add, relu_x)"
        assert (dx[x == 0] == 0).all(), f"{name}: non-zero dx where the ReLU output is 0"
    check_bf16(f"{name} dx", dx, ref["dx"], BF_FLOOR_NORM_ADD if fused else BF_FLOOR_NORM)
    if zpg is not None:
        H, W, Cc = zpg
        d4 = dx.reshape(-1, H + 1, W + 1, Cc) if rpg > 1 else dx.reshape(G, H + 1, W + 1, Cc)
        assert (d4[:, -1] == 0).all() and (d4[:, :, -1] == 0).all(), name


def norm_spg(rows, C, rpg):
    """slabs per group of vpt_norm_sums, read back from its workspace size"""
    G = rows // rpg
    return lib().vpt_norm_sums_workspace(rows, C, rpg) // (G * (2 * C + 2 * ((C // 8 + 31) // 32)))


@pytest.mark.parametrize("width", MODELS)
def test_norm_backward_at_production_shapes(width):
    s = SHAPES[width]
    N = s["N"]
    for i, (H, W, C) in enumerate(s["gn"]):  # ZP frames, many slabs per frame
        _norm_case(f"{width} GroupNorm {H}x{W}x{C} F=24", 24, (H + 1) * (W + 1), C, (H, W, C), 40 + i)
    H, W, C = s["gn"][0]  # the largest frame, with the residual and the ReLU backward in the apply pass
    _norm_case(f"{width} GroupNorm {H}x{W}x{C} F=24", 24, (H + 1) * (W + 1), C, (H, W, C), 49, fused=True)
    H, W, C = s["gn"][-1]  # the smallest frame at the production plan of whole-frame slabs
    rpg = (H + 1) * (W + 1)
    want = norm_spg(N * rpg, C, rpg)
    G = next(G for G in range(64, N + 1, 64) if norm_spg(G * rpg, C, rpg) == want)
    _norm_case(f"{width} GroupNorm {H}x{W}x{C} F={G} slabs/frame={want}", G, rpg, C, (H, W, C), 45)
    _norm_case(f"{width} GroupNorm {H}x{W}x{C} F={G} slabs/frame={want}", G, rpg, C, (H, W, C), 46, fused=True)
    for i, C in enumerate(s["ln"]):  # LayerNorm rows
        _norm_case(f"{width} LayerNorm {C}", N, 1, C, None, 50 + i)
        _norm_case(f"{width} LayerNorm {C}", N, 1, C, None, 60 + i, fused=True)
    Hf, Wf, C2, kd = s["dense"]  # the dense layer's ZP input row: rows reproducing the production column-sum plan
    want = lib().vpt_col_sums_parts(N, kd)
    rows = next(r for r in range(64, N + 1, 64) if lib().vpt_col_sums_parts(r, kd) == want)
    _norm_case(f"{width} LayerNorm dense row {kd} rows={rows}", rows, 1, kd, (Hf, Wf, C2), 55)
    nat.device_check()


# ---------------------------------------------------------------------------------------------------------------------
# max-pool, first conv, attention, softmax
# ---------------------------------------------------------------------------------------------------------------------
def unique_max_input(Fn, H, W, C, g):
    """post-ReLU pool input whose positive window maxima are unique: the 9 positions of any 3x3 window have distinct (y % 3, x % 3),
    and the value is 1 + that class + 9 * random, exact in bf16; about half the entries are 0"""
    y = torch.arange(H, device=DEV)[:, None, None] % 3
    x = torch.arange(W, device=DEV)[None, :, None] % 3
    r = torch.randint(0, 20, (Fn, H, W, C), generator=g, device=DEV)
    v = (1 + 3 * y + x + 9 * r).float()
    keep = torch.rand((Fn, H, W, C), generator=g, device=DEV) > 0.5
    return zp(torch.where(keep, v, torch.zeros((), device=DEV)) / 64)


@pytest.mark.parametrize("width", MODELS)
def test_maxpool_backward_at_production_shapes(width):
    for i, (H, W, C) in enumerate(SHAPES[width]["pools"]):
        g = gen(60 + i)
        x = unique_max_input(16, H, W, C, g)
        dy = zp(torch.randint(-128, 128, (16, H // 2, W // 2, C), generator=g, device=DEV) / 32.0)  # sums of <= 4 are exact
        out = ops.maxpool3s2_bwd(dy, x)
        ref = Rf.maxpool_bwd(dy, x).to(BF16)
        print(f"{width} maxpool bwd {H}x{W}x{C}: mismatches {(out != ref).sum().item()} (bound 0)")
        assert torch.equal(out, ref)
    nat.device_check()


def _drop_pool_near_ties(img, w, b, dy, rtol=1e-4):
    """zero dy (ZP, in place) at the pooled pixels whose two largest positive pre-pool values lie within rtol of each other (float64
    conv of the first-conv reference); returns how many"""
    C0 = w.shape[0]
    x = img.to(F64).permute(0, 3, 1, 2) / 255.0
    Wt = (w.to(F64) * 255.0).reshape(C0, 3, 3, 3).permute(0, 3, 1, 2)
    y = F.pad(F.conv2d(x, Wt, b.to(F64), padding=1).relu(), (1, 1, 1, 1), value=float("-inf"))
    top = y.unfold(2, 3, 2).unfold(3, 3, 2).reshape(*y.shape[:2], (y.shape[2] - 1) // 2, (y.shape[3] - 1) // 2, 9).topk(2, -1).values
    near = (top[..., 0] > 0) & (top[..., 0] - top[..., 1] <= rtol * top[..., 0])
    dy[:, :-1, :-1][near.permute(0, 2, 3, 1)] = 0
    return int(near.sum())


FC_C0 = sorted({SHAPES[w]["firstconv"][2] for w in WIDTHS} | {256})


@pytest.mark.parametrize("C0,f32", [(c, False) for c in FC_C0] + [(192, True), (256, True)], ids=[str(c) for c in FC_C0] + ["192-f32", "256-f32"])
def test_firstconv_backward_at_production_frames(C0, f32):
    """C0 = 256 runs the other template instance of the kernel (one 256-thread block per SM); f32: non-integer fp32 frames on the uint8
    scale, some outside [0, 255] (vpt_firstconv_bwd_f32, the pixel-gradient path)."""
    H, W = SHAPES["3x"]["firstconv"][:2]
    g = gen(70)
    if f32:
        img = torch.rand((16, H, W, 3), generator=g, device=DEV) * 340.0 - 40.0
    else:
        img = torch.randint(0, 256, (16, H, W, 3), dtype=torch.uint8, generator=g, device=DEV)
    w = randn((C0, 27), g, 0.2 / 255.0)
    b = randn((C0,), g, 0.1)
    dy = zp(randn((16, H // 2, W // 2, C0), g))
    # fp32 and float64 may pick different arg-maxima where two pooling-window values nearly tie (one such flip moves rel-L2 to ~5e-4):
    # those pooled pixels get a zero gradient, so either choice gives the same dW
    ties = _drop_pool_near_ties(img, w, b, dy)
    dW, db = ops.firstconv_bwd(img, w, b, dy, C0)
    dW_r, db_r = Rf.firstconv_bwd(img, w, b, dy)
    e_w, e_b = rel(dW / 255.0, dW_r), rel(db, db_r)
    print(f"firstconv bwd C0={C0} {'fp32' if f32 else 'u8'} frames {H}x{W} F=16 ({ties} near-tied pooling windows dropped): rel-L2 dW {e_w:.2e} "
          f"db {e_b:.2e} (bound {FC_L2:.0e})")
    assert e_w <= FC_L2 and e_b <= FC_L2
    nat.device_check()


def _attention_inputs(s, g, B=16):
    t, maxlen, heads = s["T"], s["maxlen"], s["heads"]
    h = heads * 128
    T = maxlen + t
    q = (randn((B * t, h), g) * 3).to(BF16)
    kf, vf = randn((B, T, h), g).to(BF16), randn((B, T, h), g).to(BF16)
    R = randn((B * t, heads * Rf.NBASIS), g)
    b_nd = randn((Rf.NBASIS, maxlen), g, 0.2)
    first = torch.zeros(B, t, dtype=torch.uint8, device=DEV)
    first[B // 2, 0] = 1  # a mid-batch episode start forgets its memory
    smask = (torch.rand((B, 1, maxlen), generator=g, device=DEV) > 0.3).to(torch.uint8)  # a carried-over memory
    dO = randn((B * t, h), g).to(BF16)
    return q, kf, vf, R, b_nd, first, smask, dO, B, t, maxlen, heads


@pytest.mark.parametrize("width", WIDTHS)
def test_attention_backward_at_production_shapes(width):
    s = SHAPES[width]
    args = _attention_inputs(s, gen(80))
    q, kf, vf, R, b_nd, first, smask, dO, B, t, maxlen, heads = args
    h = heads * 128
    out = torch.zeros((B * t, s["kcat"]), dtype=BF16, device=DEV)
    db = ops.attention_bwd(q, kf, vf, R, b_nd, first, smask, dO, out, B, t, maxlen, heads)
    ref = Rf.attention_bwd(*args)
    for name, sl in [("dq", slice(0, h)), ("dk", slice(h, 2 * h)), ("dv", slice(2 * h, 3 * h)), ("dR", slice(3 * h, 3 * h + heads * 10))]:
        check_bf16(f"{width} attention {heads} heads {name}", out[:, sl], ref[name], BF_FLOOR_ATTN)
    e = rel(db, ref["db_nd"])
    print(f"{width} attention d b_nd: rel-L2 {e:.2e} (bound {DBND_L2:.0e})")
    assert e <= DBND_L2
    nat.device_check()


@pytest.mark.parametrize("width", WIDTHS)
def test_softmax_backward_and_head_bias_sums(width):
    s = SHAPES[width]
    g = gen(90)
    dlog = torch.zeros((ROWS, s["ld_logits"]), dtype=BF16, device=DEV)
    scale = 1.0 / (2.0 * ROWS)
    for name, c0, n in s["head_cols"]:  # buttons: n = 8641 at the odd column 121
        logp = torch.log_softmax(randn((ROWS, n), g, 3.0), -1)
        idx = torch.randint(0, n, (ROWS,), generator=g, device=DEV)
        ops.softmax_bwd(logp, idx, scale, dlog, c0)
        check_bf16(f"{width} softmax bwd {name} n={n} col0={c0}", dlog[:, c0:c0 + n], Rf.softmax_bwd(logp, idx, scale), BF_FLOOR_SOFTMAX)
    cs = ops.col_sums(dlog)[1]  # head bias gradients
    check_sum(f"{width} col sums of d logits ({s['ld_logits']} columns)", cs, dlog.to(F64).sum(0), dlog.to(F64).abs().sum(0), DLOG_ELEM, DLOG_L2)
    nat.device_check()


def test_unmasked_attention_backward_at_idm_shapes():
    """the IDM's attention (mask "none": every key of the 128-frame sequence) at B = 4, t = 128, 32 heads, writing d q | d k | d v into
    a NaN-filled buffer with a row pitch wider than its 3h columns"""
    s = SHAPES["idm"]
    B, t, heads = s["B"], s["T"], s["heads"]
    h = heads * 128
    assert (B, t, heads, s["kcat"]) == (4, 128, 32, 3 * h)
    g = gen(85)
    q = (randn((B * t, h), g) * 3).to(BF16)
    k, v = (randn((B, t, h), g) * 3).to(BF16), randn((B, t, h), g).to(BF16)
    dO = randn((B * t, h), g).to(BF16)
    ld = s["kcat"] + 24
    ob = Guarded(B * t * ld, BF16)
    out = ob.t.view(B * t, ld)

    def call():
        ob.raw.fill_(0xFF)
        assert ops.attention_bwd(q, k, v, None, None, None, None, dO, out, B, t, 0, heads, causal=False) is None
        assert (out[:, 3 * h:].view(torch.int16) == -1).all(), "attention_bwd wrote beyond its 3h columns"
        return [out[:, :3 * h].clone()], [ob]

    _run_twice(f"idm unmasked attention_bwd B={B} t={t} heads={heads}", call)
    for i, (name, ref) in enumerate(zip(("dq", "dk", "dv"), Rf.full_attention_bwd(q, k, v, dO, B, t, heads))):
        check_bf16(f"idm attention {heads} heads {name}", out[:, i * h:(i + 1) * h], ref, BF_FLOOR_ATTN)
    nat.device_check()


def test_grouped_softmax_backward_into_the_idm_logits_gradient():
    """the IDM's factored heads (buttons 20 x 2, camera 2 x 11 classes) into their column blocks of the 64-wide logits gradient at 512
    rows, as `IDMTrainer._idm_dlog` runs them: both heads accumulate the taken sub-actions' log-probs into one `lp`; the pad columns stay
    0; then the head bias sums"""
    s = SHAPES["idm"]
    rows, ld = s["N"], s["ld_logits"]
    g = gen(95)
    dlog = torch.zeros((rows, ld), dtype=BF16, device=DEV)
    scale = 1.0 / (2.0 * rows)
    lp, lp_ref, c_end = None, torch.zeros(rows, dtype=F64, device=DEV), 0
    for name, c0, n, groups in s["head_groups"]:
        logp = torch.log_softmax(randn((rows, groups, n), g, 3.0), -1)
        idx = torch.randint(0, n, (rows, groups), generator=g, device=DEV)
        lp = ops.softmax_nll_bwd_grouped(logp, idx, scale, dlog, c0, lp=lp)
        ref = Rf.softmax_bwd(logp.reshape(rows * groups, n), idx.reshape(-1), scale).reshape(rows, groups * n)
        check_bf16(f"idm grouped softmax bwd {name} {groups}x{n} col0={c0}", dlog[:, c0:c0 + groups * n], ref, BF_FLOOR_GROUPED)
        lp_ref += logp.to(F64).gather(-1, idx[..., None]).squeeze(-1).sum(-1)
        c_end = c0 + groups * n
    assert c_end < ld and (dlog[:, c_end:] == 0).all(), "wrote into the pad columns of the logits gradient"
    e = ((lp.to(F64) - lp_ref).abs() / lp_ref.abs()).max().item()
    print(f"idm summed log-prob of the taken sub-actions: max relative error {e:.2e} (bound 8e-7)")
    assert e <= 8e-7  # measured 2.1e-7 (H100 80GB HBM3, 700 W)
    cs = ops.col_sums(dlog)[1]
    check_sum(f"idm col sums of d logits ({ld} columns)", cs, dlog.to(F64).sum(0), dlog.to(F64).abs().sum(0), DLOG_ELEM, DLOG_L2)
    nat.device_check()


# ---------------------------------------------------------------------------------------------------------------------
# writes stay inside the declared buffers; reductions are bit-reproducible
# ---------------------------------------------------------------------------------------------------------------------
PADB = 1024  # guard bytes on each side of a buffer (keeps 16-byte alignment)


class Guarded:
    """A buffer of n elements between two guard bands, all filled with 0xff bytes (a NaN in fp32 and in bf16)."""

    def __init__(self, n, dtype=F32):
        el = torch.tensor([], dtype=dtype).element_size()
        self.nb = n * el
        self.raw = torch.full((self.nb + 2 * PADB,), 0xFF, dtype=torch.uint8, device=DEV)
        self.t = self.raw[PADB:PADB + self.nb].view(dtype)

    def ptr(self):
        return self.t.data_ptr()

    def guards_intact(self):
        return bool((self.raw[:PADB] == 0xFF).all() and (self.raw[PADB + self.nb:] == 0xFF).all())


def _run_twice(name, call):
    """call() -> (outputs, guarded buffers); runs it twice, asserts untouched guards and bit-identical outputs"""
    res = []
    for _ in range(2):
        outs, bufs = call()
        torch.cuda.synchronize()
        nat.device_check()
        for i, b in enumerate(bufs):
            assert b.guards_intact(), f"{name}: write outside buffer {i}"
        res.append([o.clone() for o in outs])
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{name}: results differ between two identical calls"
    print(f"{name}: guards intact, two calls bit-identical")


def _wgrad_guarded(a, b, shifts, M_pad=8):
    R, M = a.shape
    N, nt = b.shape[1], len(shifts)
    ws_bytes = lib().vpt_wgrad_workspace_bytes(M, N, nt, R)
    ws = Guarded(max(ws_bytes, 16) // 4)
    out = Guarded((M + M_pad) * nt * N)
    sh = (C.c_int32 * nt)(*shifts)
    nat.check(lib().vpt_wgrad_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), M, N, R, sh, nt, out.ptr(), ws.ptr(), ws_bytes, stream()),
              "vpt_wgrad_bf16")
    rows = out.t.view(M + M_pad, nt * N)
    assert (rows[M:].view(torch.int32) == -1).all(), "wgrad wrote rows beyond M"
    return [rows[:M]], [ws, out]


def test_wgrad_buffers_and_determinism():
    g = gen(100)
    R = 636 * 64 + 44
    a, b = randn((R, 128), g).to(BF16), randn((R, 128), g).to(BF16)
    _run_twice("wgrad split cap", lambda: _wgrad_guarded(a, b, [0]))
    H, W, Cin, Cout = SHAPES["3x"]["convs"][0]
    dz, u = zp(randn((16, H, W, Cout), g).relu()), zp(randn((16, H, W, Cin), g))
    _run_twice("wgrad conv 3x", lambda: _wgrad_guarded(dz.view(-1, Cout), u.view(-1, Cin), conv_shifts(W)))
    M, N = SHAPES["3x"]["linears"][0]
    a, b = randn((ROWS, M), g).to(BF16), randn((ROWS, N), g).to(BF16)
    _run_twice("wgrad heads 3x", lambda: _wgrad_guarded(a, b, [0]))


def test_norm_sums_buffers_and_determinism():
    g = gen(101)
    H, W, C = SHAPES["3x"]["gn"][0]
    rpg, Fn = (H + 1) * (W + 1), 24
    x = zp(randn((Fn, H, W, C), g, 0.7, 0.3)).view(-1, C)
    du = zp(randn((Fn, H, W, C), g)).view(-1, C)
    gamma = randn((C,), g, 0.3, 1.0)
    mr = Rf.norm_stats(x, rpg, (H, W, C))
    rows, count = x.shape[0], H * W * C

    def norm_sums():
        ws, out, ms = Guarded(lib().vpt_norm_sums_workspace(rows, C, rpg)), Guarded(2 * C), Guarded(2 * Fn)
        nat.check(lib().vpt_norm_sums(du.data_ptr(), x.data_ptr(), mr.data_ptr(), gamma.data_ptr(), rows, C, rpg, float(count), out.ptr(), ms.ptr(),
                                      ws.ptr(), stream()), "vpt_norm_sums")
        dx = ops.norm_bwd_apply(du, x, mr, gamma, ms.t.view(Fn, 2), rpg, zp=(H, W, C))
        return [out.t, ms.t, dx], [ws, out, ms]

    def group_sums():
        P = lib().vpt_group_sums_parts(rpg, C)
        part, ms = Guarded(Fn * P * 2), Guarded(2 * Fn)
        nat.check(lib().vpt_group_sums(du.data_ptr(), x.data_ptr(), mr.data_ptr(), gamma.data_ptr(), part.ptr(), ms.ptr(), rows, C, rpg, float(count),
                                       stream()), "vpt_group_sums")
        return [ms.t], [part, ms]

    def col_sums(rows_, C_, du_, x_, mr_, rpg_):
        S = lib().vpt_col_sums_parts(rows_, C_)
        ws, out = Guarded(S * 2 * C_), Guarded(2 * C_)
        nat.check(lib().vpt_col_sums(du_.data_ptr(), du_.stride(0), None if x_ is None else x_.data_ptr(), None if mr_ is None else mr_.data_ptr(),
                                     rows_, C_, rpg_, out.ptr(), ws.ptr(), stream()), "vpt_col_sums")
        return [out.t], [ws, out]

    _run_twice("norm_sums + norm_bwd_apply 3x", norm_sums)
    _run_twice("group_sums 3x", group_sums)
    _run_twice("col_sums 3x frames", lambda: col_sums(rows, C, du, x, mr, rpg))
    dl = randn((ROWS, SHAPES["3x"]["ld_logits"]), g).to(BF16)
    _run_twice("col_sums d logits", lambda: col_sums(ROWS, dl.shape[1], dl, None, None, 1))


def test_pool_and_firstconv_buffers_and_determinism():
    g = gen(102)
    H, W, C = SHAPES["3x"]["pools"][0]
    Fn = 16
    x = unique_max_input(Fn, H, W, C, g)
    dy = zp(randn((Fn, H // 2, W // 2, C), g))

    def pool():
        ws, dx = Guarded(Fn * (H // 2) * (W // 2) * C // 4), Guarded(x.numel(), BF16)
        nat.check(lib().vpt_maxpool3s2_bwd(dy.data_ptr(), x.data_ptr(), dx.ptr(), ws.ptr(), Fn, H, W, C, stream()), "vpt_maxpool3s2_bwd")
        return [dx.t], [ws, dx]

    _run_twice("maxpool3s2_bwd 3x", pool)
    Hi, Wi = SHAPES["3x"]["firstconv"][:2]
    for C0 in (SHAPES["3x"]["firstconv"][2], 256):
        img = torch.randint(0, 256, (Fn, Hi, Wi, 3), dtype=torch.uint8, generator=g, device=DEV)
        w, b = randn((C0, 27), g, 0.2 / 255.0), randn((C0,), g, 0.1)
        dyf = zp(randn((Fn, Hi // 2, Wi // 2, C0), g))

        def fc():
            S = lib().vpt_firstconv_bwd_parts(Fn, Hi, Wi)
            ws, dW, db = Guarded(S * C0 * 28), Guarded(C0 * 27), Guarded(C0)
            nat.check(lib().vpt_firstconv_bwd(img.data_ptr(), w.data_ptr(), b.data_ptr(), dyf.data_ptr(), dW.ptr(), db.ptr(), ws.ptr(), Fn, Hi, Wi, C0,
                                              stream()), "vpt_firstconv_bwd")
            return [dW.t, db.t], [ws, dW, db]

        _run_twice(f"firstconv_bwd C0={C0}", fc)


def test_attention_and_softmax_buffers_and_determinism():
    s = SHAPES["3x"]
    q, kf, vf, R, b_nd, first, smask, dO, B, t, maxlen, heads = _attention_inputs(s, gen(103))
    h, ld = heads * 128, s["kcat"] + 24  # wider than the written 3h + 10 heads columns

    def attn():
        ws, out, db = Guarded(2 * B * heads * t * maxlen), Guarded(B * t * ld, BF16), Guarded(Rf.NBASIS * maxlen)
        nat.check(lib().vpt_attention_bwd(q.data_ptr(), kf.data_ptr(), vf.data_ptr(), R.data_ptr(), R.stride(0), b_nd.data_ptr(), first.data_ptr(),
                                          first.stride(0), smask.data_ptr(), dO.data_ptr(), out.ptr(), ld, db.ptr(), ws.ptr(), B, t, maxlen, heads,
                                          Rf.NBASIS, stream()), "vpt_attention_bwd")
        o = out.t.view(B * t, ld)
        assert (o[:, 3 * h + heads * Rf.NBASIS:].view(torch.int16) == -1).all(), "attention_bwd wrote beyond its columns"
        return [o[:, :3 * h + heads * Rf.NBASIS], db.t], [ws, out, db]

    _run_twice("attention_bwd 3x", attn)
    g = gen(104)
    name, c0, n = s["head_cols"][1]
    logp = torch.log_softmax(randn((ROWS, n), g, 3.0), -1)
    idx = torch.randint(0, n, (ROWS,), generator=g, device=DEV)
    ldl = s["ld_logits"]

    def smx():
        out = Guarded(ROWS * ldl, BF16)
        nat.check(lib().vpt_softmax_bwd(logp.data_ptr(), idx.data_ptr(), 0.25, out.ptr(), ldl, c0, ROWS, n, stream()), "vpt_softmax_bwd")
        o = out.t.view(ROWS, ldl)
        assert (o[:, :c0].view(torch.int16) == -1).all() and (o[:, c0 + n:].view(torch.int16) == -1).all(), "softmax_bwd wrote outside its columns"
        return [o[:, c0:c0 + n]], [out]

    _run_twice(f"softmax_bwd {name}", smx)


# ---------------------------------------------------------------------------------------------------------------------
# the whole step at 3x width
# ---------------------------------------------------------------------------------------------------------------------
def test_cuda_backward_matches_autograd_at_3x_width():
    """The forced-autograd pin of tests/test_gpu_training.py at the 3x model (perturbed weights, 128 px frames, 4 layers, 24 heads,
    B = 2): an untaped chunk fills the KV memory, then a taped chunk with a mid-batch episode start.  The same step run twice on the
    same batch gives bit-identical gradients.  T = 64 (< maxlen = 128, so the memory band is partly carried over): at T = 128 the step
    and its fp32 replica peak at 45 GiB, too much for a shared card."""
    from forced_replica import forced_loss

    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        B, T = 2, 64
        pol, sd, cfg = make_policy(vpt_b200.policy_kwargs("3x"), seed=6)
        pol = pol.to(DEV)
        g = torch.Generator().manual_seed(6)
        img0 = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).to(DEV)
        img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).to(DEV)
        actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).to(DEV), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).to(DEV)}
        first = torch.zeros(B, T, dtype=torch.bool, device=DEV)
        torch.cuda.reset_peak_memory_stats()
        (_, _, _), state = pol({"img": img0}, first, pol.initial_state(B))
        first = first.clone()
        first[1, 0] = True
        tr = BCTrainer(pol)
        tr.keep_tape = True
        loss, _ = tr.loss_and_grad(img, first, state, actions)
        grads = {n: p.grad.clone() for n, p in pol.named_parameters() if p.grad is not None}
        for p in pol.parameters():
            p.grad = None
        loss2, _ = tr.loss_and_grad(img, first, state, actions)
        nat.device_check()
        assert loss2.item() == loss.item()
        for n, p in pol.named_parameters():
            assert (p.grad is None) == (n not in grads) and (p.grad is None or torch.equal(p.grad, grads[n])), n
        del grads
        leaf = {k: v.to(DEV).clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
        lf = forced_loss(leaf, cfg, tr.last_tape, img, first, actions)
        lf.backward()
        errs = {}
        for n, p in pol.named_parameters():
            if n.startswith("value_head"):
                assert p.grad is None
                continue
            errs[n] = rel(p.grad, leaf[n].grad)
        top = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
        print(f"3x B={B} T={T}: loss {loss.item():.6f} vs forced {lf.item():.6f}; worst rel-L2 vs forced autograd: "
              + ", ".join(f"{n} {e:.4f}" for n, e in top))
        print(f"3x step: peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
        assert abs(loss.item() - lf.item()) < 1e-3 * abs(lf.item()), (loss.item(), lf.item())
        # measured at T = 128: 1.4e-2 at worst (stack-0 norms and first conv), like the small config of tests/test_gpu_training.py
        for n, e in errs.items():
            assert e < 3e-2, (n, e)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
