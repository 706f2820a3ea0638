"""The backward at the released models with the product's own weight layouts, against float64 (tests/bwd_refs.py).

1. Every input-gradient GEMM of the backward (training.py, `_gemm`: heads, lastlayer, mlp1, mlp0, proj, q | k | v | r with the residual,
   img_process.linear, dense) at the trainers' rows (2048 for BC / RL, 512 for the IDM), on the dgrad weights of the model's own
   `prepared_backward()` / `_heads_prepared_backward()`.  The reference is float64 dz @ W from the reference-schema parameter rounded to
   bf16 (as the kernel's copy is), so the bound stays at fp32-accumulation size while a layout error -- padding side, q | k | v | r
   order, the dense layer's ZP permutation, a head's column block -- is an O(1) error.  These GEMMs reach K tails the forward never
   does: K = kcat = 3h + 10 heads rounded up to 8 (the last 64-wide K tile 16 / 32 / 48 columns wide at 1x / 2x / 3x), K = 64 (the
   IDM's heads) and N up to 147 968 (the IDM's dense).  Inputs sit between NaN guard bands, outputs start 0xFF-filled, the pad columns
   of dz hold non-zero values that must not contribute, and two calls give identical bits.
2. Stack 0 of the 4x IDM at its production chunk, B x T = 4 x 128 = 512 frames, in the order `_cnn_bwd` runs it.  Its pre-pool tensor
   [512, 129, 129, 256] has more than 2^31 elements (element 2^31 lies in frame 504, byte 2^31 in frame 252).  Per-element results are
   compared on the frames around those boundaries, the sequence boundary and the last frame; the weight and norm gradients are summed
   over all 512 frames and compared against float64 sums accumulated in frame chunks.

Each check prints its measured error beside its bound, the production-chunk test its peak device memory."""
import gc

import pytest
import torch
import torch.nn.functional as F

import bwd_refs as Rf
from fwd_refs import make_model
from test_gpu_backward_shapes import (BF_FLOOR_CONV, BF_FLOOR_NORM, NORM_ELEM, NORM_L2, Guarded, _run_twice, check_bf16, check_sum,
                                      conv_shifts, wgrad_bounds)
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.training import BCTrainer, IDMTrainer, RLTrainer

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
MODELS = ["1x", "2x", "3x", "idm"]
SHAPES = {w: Rf.backward_shapes(w) for w in MODELS}

# Bounds: each is at most 4x the worst value measured on an H100 80GB HBM3 (SXM) at a 700 W power limit, given beside it.
# dgrad GEMMs: |err| <= 2^-8 |ref| + floor * (max |ref| of the row); the fp32 accumulation error grows with K: measured 1.1e-8 at K = 64
# (the IDM's heads), 1.8e-6 / 3.5e-6 / 8.1e-6 at the K tails 3152 / 6304 / 9456, 9.4e-6 at K = 16384 (the IDM's mlp0)
DGRAD_FLOOR = 3.5e-5
AFFINE_FLOOR = 2e-8    # affine_norm_zp at the production chunk; measured 5.6e-9
C3_ELEM, C3_L2 = 2.5e-9, 1.8e-7  # conv3d dW / db over 512 frames: |err| / sum |terms|, rel-L2; measured 7.3e-10, 4.5e-8
PEAK_GIB = 18          # the production-chunk test (the IDM's weights included); measured 14.8 GiB


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.fixture(scope="module", params=MODELS)
def model(request):
    """(width, shapes, policy on the device, fp32 net state dict on the CPU); one model at a time"""
    w = request.param
    pol, sd = make_model(w)
    pol = pol.to(DEV)
    m = [w, SHAPES[w], pol, sd]
    yield m
    # the policy's weight-layout caches hold it in a reference cycle (see tests/test_gpu_forward_shapes.py): free it before the next model
    m.clear()
    del pol, sd
    gc.collect()
    torch.cuda.empty_cache()
    print(f"{w} model released: {torch.cuda.memory_allocated() / 2 ** 30:.2f} GiB still allocated")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the input-gradient GEMMs
# ---------------------------------------------------------------------------------------------------------------------
def _bf(t):
    """a reference-schema parameter rounded to bf16, float64 on the device"""
    return t.detach().to(DEV).to(BF16).to(F64)


def _dense_ref_to_zp(v, Hf, Wf, C2):
    """rows in the reference's flatten order (c, y, x) -> the ZP row [(Hf+1)][(Wf+1)][C2] with a zero last row / column"""
    out = torch.zeros((v.shape[0], Hf + 1, Wf + 1, C2), dtype=v.dtype, device=v.device)
    out[:, :Hf, :Wf] = v.reshape(-1, C2, Hf, Wf).permute(0, 2, 3, 1)
    return out.reshape(v.shape[0], -1)


def _dgrad_cases(w, s, pol, sd):
    """(label, name, product dgrad weight [N][K], reference weight [K_real][N] float64 (bf16-rounded), K_real) of every dgrad GEMM"""
    wts = pol.net.prepared_backward()
    cfg = s["cfg"]
    trainers = dict(heads=IDMTrainer if w == "idm" else BCTrainer, heads_value=RLTrainer)
    for name, M, N, K, res in s["dgrads"]:
        if name in trainers:
            layers = trainers[name](pol)._head_layers()
            ref = [getattr(pol.pi_head, n).linear_layer.weight for n, _, _ in s["head_cols"]]
            if name == "heads_value":
                ref.append(pol.value_head.linear.weight)
            Wr = torch.cat([_bf(t) for t in ref])
            yield name, name, pol._heads_prepared_backward(layers), Wr, Wr.shape[0]
        elif name in ("mlp1", "mlp0", "proj", "qkvr"):
            for l in range(cfg.n_layers):
                b = f"recurrent_layer.blocks.{l}"
                o = f"{b}.r.orc_block"
                parts = ["q", "k", "v"] + (["r"] if s["causal"] else [])
                Wr = dict(mlp1=lambda: _bf(sd[f"{b}.mlp1.layer.weight"]), mlp0=lambda: _bf(sd[f"{b}.mlp0.layer.weight"]),
                          proj=lambda: _bf(sd[f"{o}.proj_layer.weight"]),
                          qkvr=lambda: torch.cat([_bf(sd[f"{o}.{c}_layer.weight"]) for c in parts]))[name]()
                yield f"{name} layer {l}", name, wts["layers"][l][name + "_t"], Wr, Wr.shape[0]
        else:
            key, p = dict(lastlayer=("last_t", "lastlayer"), linear=("linear_t", "img_process.linear"),
                          dense=("dense_t", "img_process.cnn.dense"))[name]
            Wr = _bf(sd[p + ".layer.weight"])
            yield name, name, wts[key], Wr, Wr.shape[0]


def check_rows(name, out, ref_rows, floor, step=256):
    """check_bf16 of a large bf16 [M][N] result, the float64 reference made `step` rows at a time by ref_rows(r0, r1)"""
    M = out.shape[0]
    excess, num, den, finite = -1.0, 0.0, 0.0, True
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        ref = ref_rows(r0, r1)
        o = out[r0:r1].to(F64)
        finite = finite and bool(torch.isfinite(o).all())
        rowmax = ref.abs().amax(-1, keepdim=True).clamp(min=1e-300)
        excess = max(excess, (((o - ref).abs() - 2 ** -8 * ref.abs()) / rowmax).max().item())
        num += ((o - ref) ** 2).sum().item()
        den += (ref ** 2).sum().item()
        del ref, o, rowmax
    print(f"{name}: rel-L2 {(num / den) ** 0.5:.2e}, max (|err| - 2^-8 |ref|) / row max {excess:.2e} (bound {floor:.0e})")
    assert finite and excess <= floor, name


def test_dgrad_gemms_on_the_product_layouts(model):
    w, s, pol, sd = model
    Hf, Wf, C2, _ = s["dense"]
    dims = {name: (M, N, K, res) for name, M, N, K, res in s["dgrads"]}
    seed = 0
    for label, name, Wt, Wr, kr in _dgrad_cases(w, s, pol, sd):
        M, N, K, res = dims[name]
        label = f"{w} dgrad {label} M={M} N={N} K={K} (real {kr})"
        assert tuple(Wt.shape) == (N, K) and Wt.dtype == BF16 and Wt.is_contiguous(), (label, tuple(Wt.shape))
        seed += 1
        g = gen(seed)
        db = Guarded(M * K, BF16)
        dz = db.t.view(M, K)
        dz.copy_(torch.randn((M, K), generator=g, device=DEV).to(BF16))  # pad columns [kr, K) too: they must not contribute
        bufs = [db]
        resid = None
        if res:
            rb = Guarded(M * N, BF16)
            resid = rb.t.view(M, N)
            resid.copy_(torch.randn((M, N), generator=g, device=DEV).to(BF16))
            bufs.append(rb)
        ob = Guarded(M * N, BF16)
        out = ob.t.view(M, N)

        def call():
            ob.raw.fill_(0xFF)
            ops.gemm(dz, Wt, out, M, N, K, residual=resid)
            return [out.clone()], bufs + [ob]

        _run_twice(label, call)
        if name == "dense":  # the ZP pad row / column of the CNN output gets exactly 0
            o4 = out.view(M, Hf + 1, Wf + 1, C2)
            assert (o4[:, -1] == 0).all() and (o4[:, :, -1] == 0).all(), f"{label}: non-zero gradient in the ZP pad row / column"

            def ref_rows(r0, r1):
                return _dense_ref_to_zp(dz[r0:r1, :kr].to(F64) @ Wr, Hf, Wf, C2)
        else:
            def ref_rows(r0, r1):
                r = dz[r0:r1, :kr].to(F64) @ Wr
                return r if resid is None else r + resid[r0:r1].to(F64)

        check_rows(label, out, ref_rows, DGRAD_FLOOR)
        del dz, db, ob, out, resid, bufs
    nat.device_check()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the IDM's stack 0 at the production chunk
# ---------------------------------------------------------------------------------------------------------------------
FRAMES = [0, 127, 128, 252, 503, 504, 505, 511]  # sequence ends, byte 2^31 and element 2^31 of [512, 129, 129, 256], the last frame


def _fill_zp(shape, g, fn, step=16):
    """bf16 ZP frames [F, H+1, W+1, C] with zero pads, the interior made by fn(frames, generator) [n, H, W, C] `step` frames at a time"""
    Fn, Hp, Wp, Cc = shape
    t = torch.zeros(shape, dtype=BF16, device=DEV)
    for f0 in range(0, Fn, step):
        f1 = min(Fn, f0 + step)
        t[f0:f1, :-1, :-1] = fn(f1 - f0, g).to(BF16)
    return t


def _unique_max(n, H, W, C, g):
    """the interior of test_gpu_backward_shapes.unique_max_input: positive window maxima unique, exact in bf16, about half zeros"""
    y = torch.arange(H, device=DEV)[:, None, None] % 3
    x = torch.arange(W, device=DEV)[None, :, None] % 3
    v = (1 + 3 * y + x + 9 * torch.randint(0, 20, (n, H, W, C), generator=g, device=DEV)).float()
    keep = torch.rand((n, H, W, C), generator=g, device=DEV) > 0.5
    return torch.where(keep, v, torch.zeros((), device=DEV)) / 64


def _chunked(Fn, fn, step=16):
    """sum over frame chunks of the tuple fn(f0, f1)"""
    acc = None
    for f0 in range(0, Fn, step):
        r = fn(f0, min(Fn, f0 + step))
        acc = list(r) if acc is None else [a + b for a, b in zip(acc, r)]
    return acc


def test_idm_stack0_backward_at_the_production_chunk(model):
    """`_cnn_bwd` on stack 0 of the 4x IDM at 512 frames: max-pool backward, the dgrad conv on the product's
    prepared_backward()["stacks"][0]["first"], affine_norm_zp and the wgrad with the nine ZP shifts over all 8.5 M rows, norm_sums +
    norm_bwd_apply(relu_x) on the conv3d output, and conv3d_t5_bwd on uint8 and on non-integer fp32 frames"""
    w, s, pol, sd = model
    if w != "idm":
        pytest.skip("the policies' stack 0 is the fused first conv (test_gpu_backward_shapes.py: test_firstconv_backward_at_production_frames)")
    B, T = s["B"], s["T"]
    Fn = B * T
    H, W, Cin, C = s["convs"][0]
    assert (Fn, Cin, C) == (512, 128, 256) and s["pools"][0] == (H, W, C) and s["gn"][0] == (H, W, Cin)
    P = (H + 1) * (W + 1)
    R = Fn * P
    assert R * C > 2 ** 31 and R * Cin < 2 ** 31 < R * Cin * 2
    p = "img_process.cnn.stacks.0.firstconv"
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    g = gen(500)
    # 1. ReLU -> max-pool backward into the pre-pool gradient
    x_full = _fill_zp((Fn, H + 1, W + 1, C), g, lambda n, gg: _unique_max(n, H, W, C, gg))
    dy1 = _fill_zp((Fn, H // 2 + 1, W // 2 + 1, C), g,
                   lambda n, gg: torch.randint(-128, 128, (n, H // 2, W // 2, C), generator=gg, device=DEV) / 32.0, step=64)
    dfull = ops.maxpool3s2_bwd(dy1, x_full)
    ref = Rf.maxpool_bwd(dy1[FRAMES], x_full[FRAMES]).to(BF16)
    bad = (dfull[FRAMES] != ref).sum().item()
    print(f"idm stack 0 maxpool bwd {H}x{W}x{C} F={Fn} frames {FRAMES}: mismatches {bad} (bound 0)")
    assert bad == 0
    del x_full, dy1, ref
    # 2. the dgrad conv on the product's rotated weight, against conv2d_input with the reference-schema weight
    Wrot = pol.net.prepared_backward()["stacks"][0]["first"]
    Wt = sd[p + ".layer.weight"].to(DEV).to(BF16)
    du, _ = ops.conv3x3_zp(dfull, Wrot, H, W, relu=0, want_stats=False)
    assert (du[FRAMES][:, -1] == 0).all() and (du[FRAMES][:, :, -1] == 0).all()
    ref, _ = Rf.conv_dgrad(dfull[FRAMES], Wt)
    check_bf16(f"idm stack 0 dgrad conv {C}->{Cin} F={Fn} frames {FRAMES}", du[FRAMES], ref, BF_FLOOR_CONV)
    del ref
    # 3. the conv3d output (post-ReLU) and its GroupNorm: affine_norm_zp -> u, the wgrad over all rows
    x_in = _fill_zp((Fn, H + 1, W + 1, Cin), g, lambda n, gg: torch.randn((n, H, W, Cin), generator=gg, device=DEV).relu())
    mr = torch.cat([Rf.norm_stats(x_in[f0:f0 + 16].view(-1, Cin), P, (H, W, Cin)) for f0 in range(0, Fn, 16)])
    gam = sd[p + ".norm.weight"].to(DEV).float().contiguous()
    bet = sd[p + ".norm.bias"].to(DEV).float().contiguous()
    u, _ = ops.affine_norm_zp(x_in, mr, gam, bet)
    ref = Rf.to_zp(F.group_norm(Rf.nchw(x_in[FRAMES]), 1, gam.to(F64), bet.to(F64), eps=1e-5))
    check_bf16(f"idm stack 0 affine_norm_zp {H}x{W}x{Cin} F={Fn} frames {FRAMES}", u[FRAMES], ref, AFFINE_FLOOR)
    del ref
    dW = ops.wgrad(dfull.view(R, C), u.view(R, Cin), conv_shifts(W))
    ref, scale = _chunked(Fn, lambda f0, f1: Rf.conv_wgrad_taps(dfull[f0:f1], u[f0:f1]), step=8)
    check_sum(f"idm stack 0 wgrad {C}x9x{Cin} over R={R} rows", dW, ref, scale, *wgrad_bounds(C, Cin, 9, R))
    del dfull, u, dW, ref, scale
    # 4. the norm's backward with the conv3d's ReLU backward fused (relu_x): dgamma / dbeta / per-frame sums over all frames, dx per frame
    cs, ms = ops.norm_sums(du.view(R, Cin), x_in.view(R, Cin), mr, gam, P, H * W * Cin)

    def norm_chunk(f0, f1):
        d, x = du[f0:f1].view(-1, Cin), x_in[f0:f1].view(-1, Cin)
        r = Rf.norm_bwd(d, x, gam, P, (H, W, Cin))
        grp = torch.arange(x.shape[0], device=DEV) // P
        n = ((x.to(F64) - mr[f0:f1][grp, 0:1].to(F64)) * mr[f0:f1][grp, 1:2].to(F64)).abs()
        a = d.to(F64).abs()
        return r["dgamma"], r["dbeta"], (a * n).sum(0), a.sum(0)

    dg, dbt, sg, sbt = _chunked(Fn, norm_chunk, step=8)
    check_sum(f"idm stack 0 norm dgamma over {Fn} frames", cs[0], dg, sg, NORM_ELEM, NORM_L2)
    check_sum(f"idm stack 0 norm dbeta over {Fn} frames", cs[1], dbt, sbt, NORM_ELEM, NORM_L2)
    ref = Rf.norm_bwd(du[FRAMES].view(-1, Cin), x_in[FRAMES].view(-1, Cin), gam, P, (H, W, Cin), relu_x=True)
    d, x = du[FRAMES].view(len(FRAMES), -1, Cin).to(F64), x_in[FRAMES].view(len(FRAMES), -1, Cin).to(F64)
    gdu = (d * gam.to(F64)).abs()
    n = ((x - mr[FRAMES, 0, None, None].to(F64)) * mr[FRAMES, 1, None, None].to(F64)).abs()
    ms_scale = torch.stack([gdu.sum((1, 2)), (gdu * n).sum((1, 2))], 1) / (H * W * Cin)
    del d, x, gdu, n
    check_sum(f"idm stack 0 norm per-frame sums, frames {FRAMES}", ms[FRAMES], ref["ms"], ms_scale, NORM_ELEM, NORM_L2)
    dx = ops.norm_bwd_apply(du.view(R, Cin), x_in.view(R, Cin), mr, gam, ms, P, zp=(H, W, Cin), relu_x=True).view(Fn, H + 1, W + 1, Cin)
    del du, cs, ms
    sel = dx[FRAMES]
    assert (sel[x_in[FRAMES] == 0] == 0).all(), "norm_bwd_apply(relu_x): non-zero gradient where the ReLU output is 0"
    check_bf16(f"idm stack 0 norm dx (relu_x) F={Fn} frames {FRAMES}", sel.view(-1, Cin), ref["dx"], BF_FLOOR_NORM)
    del ref, sel
    # 5. conv3d_t5_bwd on uint8 and on non-integer fp32 frames
    frames = {"u8": torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g, device=DEV),
              "f32": torch.rand((B, T, H, W, 3), generator=g, device=DEV) * 340.0 - 40.0}
    for kind, img in frames.items():
        dW3, db3 = ops.conv3d_t5_bwd(img, dx, Cin)
        rW, rb, sW, sb = Rf.conv3d_t5_wgrad(img, dx, Cin)
        check_sum(f"idm conv3d_t5_bwd dW ({kind} frames) over {Fn} frames", dW3, rW, sW, C3_ELEM, C3_L2)
        check_sum(f"idm conv3d_t5_bwd db ({kind} frames) over {Fn} frames", db3, rb, sb, C3_ELEM, C3_L2)
    del dx, x_in, frames
    nat.device_check()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"idm stack 0 at {Fn} frames: peak device memory {peak:.1f} GiB (bound {PEAK_GIB})")
    assert peak <= PEAK_GIB
