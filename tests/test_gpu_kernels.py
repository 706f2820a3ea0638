"""GPU: every C-ABI entry point against the torch emulation of the same op (tests/emu_ops.py, CPU fp32), i.e. against the
arithmetic the oracle uses.  Integer / index results must be bit exact; bf16 results within bf16 rounding of fp32 math."""
import pytest
import torch

import emu_ops as E
import vpt_b200
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _close(name, got, ref, rtol=2e-2, atol=2e-2, l2=4e-3):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    err = (got - ref).abs()
    rel = (got - ref).norm() / ref.norm().clamp(min=1e-20)
    bad = err > atol + rtol * ref.abs()
    assert not bad.any() and rel < l2, (f"{name}: {int(bad.sum())}/{bad.numel()} elements out of tolerance, max abs err {err.max():.4g}, "
                                        f"rel l2 {rel:.3g}; first bad idx {bad.nonzero()[:4].tolist()}; got {got[bad][:4].tolist()} ref {ref[bad][:4].tolist()}")


def _rand(shape, g, scale=1.0, dtype=BF16):
    return (torch.randn(shape, generator=g) * scale).to(dtype)


def _gemm_case(M, N, K, g, *, conv=None, fold=False, relu=0, residual=None, out_f32=False, out_scale=1.0, seg=None, stats=0, bias=False):
    if conv is not None:
        H, W, Cin = conv
        A = _rand((M // (H * W), H, W, Cin), g)
        ncls = 9
    else:
        A = _rand((M, K), g)
        ncls = 1
    Bw = _rand((N, K), g, K ** -0.5)
    mr = S1 = S2 = None
    rpg = (conv[0] * conv[1]) if conv is not None else 1
    if fold:
        G = M // rpg
        mr = torch.stack([torch.randn(G, generator=g) * 0.3, torch.rand(G, generator=g) + 0.5], 1)
        S1 = torch.randn(ncls, N, generator=g)
        S2 = torch.randn(ncls, N, generator=g)
    elif bias:
        S2 = torch.randn(ncls, N, generator=g)
    res = None
    if residual is not None:
        res = _rand((M, N), g, dtype=residual)
    rows_out = M if seg is None else (M // seg[0]) * seg[1]
    odt = F32 if out_f32 else BF16
    P = E.gemm_stat_parts(N)
    assert P == ops.gemm_stat_parts(N)
    srows = M if stats == 1 else (M + 31) // 32

    def run(mod, dev, cluster=0):
        out = torch.zeros((rows_out, N), dtype=odt, device=dev)
        part = torch.zeros((srows, P, 2), dtype=F32, device=dev) if stats else None
        to = lambda t: None if t is None else t.to(dev)
        mod.gemm(to(A), to(Bw), out, M, N, K, conv=conv, mr=to(mr), rows_per_group=rpg, S1=to(S1), S2=to(S2), relu=relu, out_scale=out_scale,
                 residual=to(res), seg=seg, stat_part=part, stat_mode=stats, cluster=cluster)
        st = None
        if stats:
            npg = (rpg // 32 if stats == 2 else rpg) * P
            st = mod.stats_finalize(part, M // rpg, npg, rpg * N)
        return out, st

    ref, rst = run(E, "cpu")
    for cluster in (1, 2, 4):  # CTAs per cluster sharing the B tile by TMA multicast
        got, gst = run(ops, DEV, cluster)
        nat.device_check()
        _close(f"gemm M={M} N={N} K={K} conv={conv} fold={fold} cluster={cluster}", got, ref)
        if stats:
            _close(f"gemm stats cluster={cluster}", gst, rst, rtol=2e-3, atol=2e-3, l2=1e-3)


def test_gemm_small_m_weight_streaming_path():
    """M <= 8 rows take csrc/gemv_small.cuh (rollout path); same contract as the tensor-core kernel, incl. stats and row remap."""
    g = torch.Generator().manual_seed(21)
    for M in (1, 3, 8):
        _gemm_case(M, 2048, 2048, g, bias=True, stats=1)
        _gemm_case(M, 256, 73984, g, fold=True, relu=1, stats=1)
        _gemm_case(M, 8762, 256, g, bias=True, out_f32=True, out_scale=0.5)
        _gemm_case(M, 512, 256, g, bias=True, residual=BF16, relu=2, stats=1)
    _gemm_case(4, 256, 256, g, seg=(2, 6, 4))
    _gemm_case(1, 1, 2048, g, bias=True, out_f32=True)
    try:  # and the tensor-core kernel on the same tiny shapes
        nat.lib().vpt_debug_set(0, -1)
        _gemm_case(3, 2048, 2048, g, bias=True, stats=1)
    finally:
        nat.lib().vpt_debug_set(0, 0)


def test_gemm_linear_plain():
    g = torch.Generator().manual_seed(0)
    _gemm_case(128, 128, 64, g)
    _gemm_case(256, 256, 256, g)
    _gemm_case(300, 200, 192, g)        # ragged M and N


def test_gemm_linear_multi_tile_long_k():
    g = torch.Generator().manual_seed(1)
    _gemm_case(1000, 2048, 2048, g, bias=True)           # 8 x 8 tiles, pipeline wraps many times
    _gemm_case(20000, 256, 512, g, bias=True, relu=1)     # more tiles than SMs: persistent loop + staging-tile reuse


def test_gemm_partial_last_k_tile():
    """K = 3h + 10 heads rounded up to 8, the q | k | v | r dgrad GEMM of the backward with its residual at the 1x / 2x / 3x widths: the
    last 64-wide K tile is 16, 32 and 48 columns wide.  K = 64: one K tile (the IDM's heads dgrad)."""
    g = torch.Generator().manual_seed(5)
    for K in (3152, 6304, 9456):
        assert K % 64 in (16, 32, 48)
        _gemm_case(256, 512, K, g, residual=BF16)
    _gemm_case(512, 1024, 64, g)
    _gemm_case(300, 200, 64, g, residual=BF16)


def test_gemm_linear_epilogues():
    g = torch.Generator().manual_seed(2)
    _gemm_case(384, 512, 256, g, fold=True, relu=1, stats=1)
    _gemm_case(384, 512, 256, g, bias=True, residual=BF16, stats=1)
    _gemm_case(384, 512, 256, g, bias=True, residual=BF16, relu=2, stats=1)
    _gemm_case(384, 160, 256, g, bias=True, out_f32=True)
    _gemm_case(96, 8763, 256, g, bias=True, out_f32=True, out_scale=0.5)   # heads: ragged N, unaligned ld handled by caller
    _gemm_case(96, 1, 256, g, bias=True, out_f32=True)
    _gemm_case(64, 256, 256, g, seg=(8, 24, 16))                            # KV row remap: (b, i) -> b*24 + 16 + i


@pytest.mark.parametrize("H,W,Cin,Cout,F_", [(16, 16, 64, 64, 3), (8, 8, 128, 128, 5), (4, 4, 128, 128, 11), (32, 32, 128, 256, 2),
                                             (64, 64, 128, 128, 2), (16, 16, 256, 256, 3), (32, 32, 192, 384, 1)])
def test_gemm_conv3x3(H, W, Cin, Cout, F_):
    g = torch.Generator().manual_seed(3)
    mode = 2 if (H * W) % 32 == 0 else 1
    _gemm_case(F_ * H * W, Cout, 9 * Cin, g, conv=(H, W, Cin), fold=True, relu=1, stats=mode)
    _gemm_case(F_ * H * W, Cout, 9 * Cin, g, conv=(H, W, Cin), fold=True, relu=1, residual=BF16, stats=mode)


@pytest.mark.parametrize("H,W,Cin,Cout,F_", [(16, 16, 64, 64, 3), (8, 8, 128, 128, 120), (4, 4, 128, 128, 11), (4, 4, 128, 128, 400), (32, 32, 128, 256, 2),
                                             (64, 64, 128, 128, 3), (64, 64, 128, 128, 1), (64, 64, 128, 256, 1), (16, 16, 256, 256, 3), (32, 32, 192, 384, 1),
                                             (32, 32, 256, 256, 7), (16, 16, 128, 128, 40), (16, 16, 128, 128, 2), (32, 32, 256, 256, 1), (16, 16, 256, 256, 1),
                                             (64, 64, 128, 256, 1), (32, 32, 192, 384, 1)])
def test_conv3x3_zp(H, W, Cin, Cout, F_):
    """ZP-layout conv with the input span reused across the 9 taps (shifted wgmma descriptors) vs F.conv2d + fold."""
    g = torch.Generator().manual_seed(13)
    x = E.to_zp(_rand((F_, H, W, Cin), g))
    Wb = _rand((Cout, 9 * Cin), g, (9 * Cin) ** -0.5)
    mr = torch.stack([torch.randn(F_, generator=g) * 0.3, torch.rand(F_, generator=g) + 0.5], 1)
    S1, S2 = torch.randn(9, Cout, generator=g), torch.randn(9, Cout, generator=g)
    res = E.to_zp(_rand((F_, H, W, Cout), g))
    try:
        # every value of the kernel-choice knobs must give the same results (this build has one convolution kernel for all of them)
        for pair, swap in ((0, 0), (2, 0), (0, 1), (0, 4), (0, 5)) if Cout == 128 else ((0, 0), (2, 0), (0x100, 0), (0x102, 0)):
            nat.lib().vpt_set_conv_pair_mode(pair)
            nat.lib().vpt_set_conv_swap_mode(swap)
            for residual in (None, res):
                got, gmr = ops.conv3x3_zp(x.to(DEV), Wb.to(DEV), H, W, mr=mr.to(DEV), S1=S1.to(DEV), S2=S2.to(DEV), relu=1,
                                          residual=None if residual is None else residual.to(DEV))
                nat.device_check()
                ref, rmr = E.conv3x3_zp(x, Wb, H, W, mr=mr, S1=S1, S2=S2, relu=1, residual=residual)
                gc = got.cpu()
                assert (gc[:, -1] == 0).all() and (gc[:, :, -1] == 0).all(), "ZP zero row/column not maintained by the conv epilogue"
                _close(f"conv3x3_zp pair={pair} swap={swap} {F_}x{H}x{W} {Cin}->{Cout} res={residual is not None}", got, ref)
                _close(f"conv3x3_zp stats pair={pair} swap={swap}", gmr, rmr, rtol=2e-3, atol=2e-3, l2=1e-3)
    finally:
        nat.lib().vpt_set_conv_pair_mode(1)
        nat.lib().vpt_set_conv_swap_mode(1)


def test_zp_pool_norm():
    g = torch.Generator().manual_seed(14)
    x = E.to_zp(_rand((3, 16, 16, 128), g).relu())
    got, gmr = ops.maxpool3s2(x.to(DEV), zp=True)
    ref, rmr = E.maxpool3s2(x, zp=True)
    assert torch.equal(got.cpu(), ref), "ZP maxpool must be bit exact (incl. zero row/column)"
    _close("zp pool stats", gmr, rmr, rtol=1e-3, atol=1e-3, l2=1e-3)
    gam, bet = torch.randn(128, generator=g), torch.randn(128, generator=g)
    got2, gmr2 = ops.affine_norm_zp(ref.to(DEV), rmr.to(DEV), gam.to(DEV), bet.to(DEV))
    ref2, rmr2 = E.affine_norm_zp(ref, rmr, gam, bet)
    nat.device_check()
    g2 = got2.cpu()
    assert (g2[:, -1] == 0).all() and (g2[:, :, -1] == 0).all()
    _close("affine_norm_zp", got2, ref2, rtol=1e-2, atol=1e-2)
    _close("affine_norm_zp stats", gmr2, rmr2, rtol=2e-3, atol=2e-3, l2=1e-3)


def test_firstconv_pool():
    g = torch.Generator().manual_seed(4)
    for (F_, H, W, C0) in [(3, 32, 32, 64), (2, 128, 128, 128), (1, 64, 64, 192)]:
        img = torch.randint(0, 256, (F_, H, W, 3), dtype=torch.uint8, generator=g)
        w = torch.randn(C0, 27, generator=g) / 255.0 * 0.3
        b = torch.randn(C0, generator=g) * 0.1
        for zp in (True, False):
            got, gmr = ops.firstconv_pool(img.to(DEV), w.to(DEV), b.to(DEV), C0, zp=zp)
            nat.device_check()
            ref, rmr = E.firstconv_pool(img, w, b, C0, zp=zp)
            _close(f"firstconv_pool {F_}x{H}x{W}x{C0} zp={zp}", got, ref, rtol=1e-2, atol=1e-3, l2=3e-3)
            _close("firstconv stats", gmr, rmr, rtol=2e-3, atol=2e-3, l2=1e-3)
            if zp:
                gc = got.cpu()
                assert (gc[:, -1] == 0).all() and (gc[:, :, -1] == 0).all()


def test_maxpool_and_affine_norm():
    g = torch.Generator().manual_seed(5)
    x = _rand((3, 16, 16, 128), g).relu()
    got, gmr = ops.maxpool3s2(x.to(DEV), zp=False)
    ref, rmr = E.maxpool3s2(x, zp=False)
    assert torch.equal(got.cpu(), ref), "maxpool must be bit exact"
    _close("pool stats", gmr, rmr, rtol=1e-3, atol=1e-3, l2=1e-3)
    gam, bet = torch.randn(128, generator=g), torch.randn(128, generator=g)
    for rpg in (64, 1):
        xr = ref.reshape(-1, 128)
        mr = E._row_stats(xr, rpg)
        got2, g32, gmr2 = ops.affine_norm(xr.to(DEV), mr.to(DEV), gam.to(DEV), bet.to(DEV), rpg, want_stats=True, want_f32=True)
        ref2, r32, rmr2 = E.affine_norm(xr, mr, gam, bet, rpg, want_stats=True, want_f32=True)
        nat.device_check()
        _close("affine_norm bf16", got2, ref2, rtol=1e-2, atol=1e-2)
        _close("affine_norm f32", g32, r32, rtol=1e-4, atol=1e-4, l2=1e-5)
        _close("affine_norm stats", gmr2, rmr2, rtol=2e-3, atol=2e-3, l2=1e-3)


def test_copy_rows_and_state_mask():
    g = torch.Generator().manual_seed(6)
    src = torch.randn(3, 10, 256, generator=g)
    dst_g = torch.zeros(3, 14, 256, dtype=BF16, device=DEV)
    dst_r = torch.zeros(3, 14, 256, dtype=BF16)
    ops.copy_rows(src.to(DEV), 2, dst_g, 5, 7)
    E.copy_rows(src, 2, dst_r, 5, 7)
    assert torch.equal(dst_g.cpu(), dst_r)
    back_g = torch.zeros(3, 7, 256, device=DEV)
    ops.copy_rows(dst_g, 5, back_g, 0, 7)
    assert torch.equal(back_g.cpu(), dst_r[:, 5:12].float())
    for t, maxlen in [(3, 8), (8, 8), (20, 8), (1, 128)]:
        first = torch.zeros(4, t, dtype=torch.bool)
        first[2, 0] = True
        mask = (torch.rand(4, 1, maxlen, generator=g) > 0.5)
        for m in (None, mask):
            got = ops.state_mask_update(None if m is None else m.to(DEV).view(torch.uint8), first.to(DEV).view(torch.uint8), t, maxlen)
            ref = E.state_mask_update(None if m is None else m.view(torch.uint8), first.view(torch.uint8), t, maxlen)
            assert torch.equal(got.cpu(), ref), (t, maxlen)
    nat.device_check()


@pytest.mark.parametrize("B,t,maxlen,heads", [(2, 8, 8, 2), (3, 128, 128, 2), (2, 1, 128, 3), (1, 77, 128, 1), (2, 200, 128, 2), (2, 5, 16, 2)])
def test_attention(B, t, maxlen, heads):
    g = torch.Generator().manual_seed(7)
    h = heads * 128
    T = maxlen + t
    Q, Kf, Vf = _rand((B, t, h), g, 3.0), _rand((B, T, h), g, 3.0), _rand((B, T, h), g)
    R = torch.randn(B, t, heads * 10, generator=g)
    b_nd = torch.randn(10, maxlen, generator=g) * 0.5
    first = torch.zeros(B, t, dtype=torch.bool)
    first[B - 1, 0] = True
    smask = (torch.rand(B, 1, maxlen, generator=g) > 0.3)
    for sm in (None, smask):
        got = ops.attention(Q.to(DEV), Kf.to(DEV), Vf.to(DEV), R.to(DEV), b_nd.to(DEV), first.to(DEV).view(torch.uint8),
                            None if sm is None else sm.to(DEV).view(torch.uint8), B, t, maxlen, heads)
        nat.device_check()
        ref = E.attention(Q, Kf, Vf, R, b_nd, first.view(torch.uint8), None if sm is None else sm.view(torch.uint8), B, t, maxlen, heads)
        _close(f"attention smask={'yes' if sm is not None else 'none'}", got, ref, rtol=2e-2, atol=2e-2, l2=6e-3)


def test_attention_unmasked_idm():
    g = torch.Generator().manual_seed(8)
    B, t, heads = 2, 128, 2
    h = heads * 128
    Q, Kf, Vf = _rand((B, t, h), g, 3.0), _rand((B, t, h), g, 3.0), _rand((B, t, h), g)
    got = ops.attention(Q.to(DEV), Kf.to(DEV), Vf.to(DEV), None, None, None, None, B, t, 0, heads, causal=False)
    nat.device_check()
    ref = E.attention(Q, Kf, Vf, None, None, None, None, B, t, 0, heads, causal=False)
    _close("attention unmasked", got, ref, rtol=2e-2, atol=2e-2, l2=6e-3)


def test_heads_tail():
    g = torch.Generator().manual_seed(9)
    rows, ld = 37, 8768
    raw = torch.randn(rows, ld, generator=g) * 3
    for c0, n in [(0, 121), (121, 8641)]:
        got = ops.log_softmax(raw.to(DEV), c0, n)
        ref = E.log_softmax(raw, c0, n)
        _close("log_softmax", got, ref, rtol=1e-5, atol=2e-5, l2=1e-5)
    lg = E.log_softmax(raw, 121, 8641)
    u = torch.rand(rows, 8641, generator=g)
    u[0, 5] = 1.0
    # (1) vs torch's own CUDA ops on identical inputs (what the reference would execute on this GPU): bit exact
    lg_d, u_d = lg.to(DEV), u.to(DEV)
    got = ops.gumbel_argmax(lg_d, u_d)
    u2 = u_d.clone()
    u2[u2 == 1.0] = 0.999
    ref_d = torch.argmax(lg_d - torch.log(-torch.log(u2)), dim=-1)
    assert torch.equal(got, ref_d), "Gumbel-max sampling differs from torch CUDA ops on identical logits+uniforms"
    # (2) vs the CPU oracle formula (libm vs CUDA logf may differ in the last ulp -> report, require near-total agreement)
    ref_c = E.gumbel_argmax(lg, u)
    assert (got.cpu() == ref_c).float().mean() >= 0.97
    assert torch.equal(ops.gumbel_argmax(lg_d, None).cpu(), torch.argmax(lg, -1))
    # ties -> lowest index
    tie = torch.zeros(4, 100)
    tie[:, [7, 50]] = 1.0
    assert ops.gumbel_argmax(tie.to(DEV), None).tolist() == [7, 7, 7, 7]
    lp = ops.gather_logprob(lg_d, got)
    assert torch.equal(lp.cpu(), lg.gather(-1, got.cpu().unsqueeze(-1)).squeeze(-1))
    nat.device_check()


def test_fused_adam_matches_torch_optim():
    """vpt_adam_step over a flat bucket vs torch.optim.Adam(lr, weight_decay) (behavioural_cloning.py:63-67), 5 steps."""
    from video_pre_training_b200.parallel import FlatAdamDP
    g = torch.Generator().manual_seed(31)
    shapes = [(257, 33), (1001,), (64, 3, 3, 3), (7,)]
    ref_params = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in shapes]
    our_params = [torch.nn.Parameter(p.detach().clone().to(DEV)) for p in ref_params]
    ref = torch.optim.Adam(ref_params, lr=1.81e-4, weight_decay=0.039428)
    ours = FlatAdamDP(our_params, lr=1.81e-4, weight_decay=0.039428)
    for step in range(5):
        grads = [torch.randn(s, generator=g) for s in shapes]
        ours.zero_grad()
        for p, q, gr in zip(ref_params, our_params, grads):
            p.grad = gr.clone()
            q.grad.copy_(gr.to(DEV))          # .grad aliases the flat gradient bucket
        ref.step()
        ours.step()
    nat.device_check()
    for p, q in zip(ref_params, our_params):
        assert torch.allclose(q.detach().cpu(), p.detach(), rtol=1e-5, atol=1e-7), (q.detach().cpu() - p.detach()).abs().max()


def test_gemm_column_segments_fused_qkvr():
    """vpt_gemm_args.dst_*: ONE GEMM over the concatenated Q | K | V | R weight writes each column segment to its own destination
    (bf16 q; K / V into the rows after the memory of the [B][maxlen + t][h] buffers through the row remap; R in fp32) == four GEMMs."""
    g = torch.Generator().manual_seed(31)
    for (B, t, maxlen, h, heads) in [(3, 8, 16, 256, 2), (2, 128, 128, 1024, 8), (1, 1, 16, 256, 2), (4, 2, 128, 1024, 8)]:  # last two: the small-M weight-streaming kernel
        M, T, nr = B * t, maxlen + t, 10 * heads
        x = _rand((M, h), g)
        Wc = _rand((3 * h + nr, h), g, h ** -0.5)
        bias = torch.randn(3 * h + nr, generator=g)

        def run(mod, dev):
            to = lambda v: v.to(dev)
            q = torch.zeros((M, h), dtype=BF16, device=dev)
            fk = torch.zeros((B, T, h), dtype=BF16, device=dev)
            fv = torch.zeros((B, T, h), dtype=BF16, device=dev)
            R = torch.zeros((M, nr), dtype=F32, device=dev)
            mod.gemm(to(x), to(Wc), q, M, 3 * h + nr, h, S2=to(bias), seg=(t, T, maxlen),
                     dsts=[(0, q, h, False), (h, fk, h, True), (2 * h, fv, h, True), (3 * h, R, nr, False)])
            return q, fk, fv, R

        ref = run(E, "cpu")
        got = run(ops, DEV)
        nat.device_check()
        for name, a, b in zip("q k v R".split(), got, ref):
            _close(f"fused qkvr {name} B={B} t={t} h={h}", a, b)
        assert (got[1][:, :maxlen] == 0).all() and (got[2][:, :maxlen] == 0).all(), "memory rows must not be touched"


def test_two_norm_composition_kernels():
    """vpt_norm2_fold + the Ef / res_scale modes of vpt_conv3x3_zp (every epilogue: SM pairs with TMA store, single CTA, operand-swapped)
    + the per-channel partials of vpt_maxpool3s2 / vpt_firstconv_pool, each against the test-only emulation."""
    g = torch.Generator().manual_seed(41)
    # per-channel partials of the two pool producers
    x = E.to_zp(_rand((3, 16, 16, 256), g).relu())
    got, gmr, gch = ops.maxpool3s2(x.to(DEV), zp=True, want_chan=True)
    ref, rmr, rch = E.maxpool3s2(x, zp=True, want_chan=True)
    assert torch.equal(got.cpu(), ref)
    _close("maxpool per-channel sums", gch.sum(1), rch.sum(1), rtol=1e-4, atol=1e-3)
    img = torch.randint(0, 256, (2, 64, 64, 3), dtype=torch.uint8, generator=g)
    w = torch.randn(128, 27, generator=g) / 255.0 * 0.3
    b = torch.randn(128, generator=g) * 0.1
    _, _, gch = ops.firstconv_pool(img.to(DEV), w.to(DEV), b.to(DEV), 128, zp=True, want_chan=True)
    _, _, rch = E.firstconv_pool(img, w, b, 128, zp=True, want_chan=True)
    _close("firstconv per-channel sums", gch.sum(1), rch.sum(1), rtol=2e-3, atol=5e-2)
    # fold tables
    F_, C, Cout = 5, 128, 128
    chan = torch.rand(F_, 7, C, 2, generator=g) * 50 + 20
    chan[..., 1] += chan[..., 0] ** 2 / 10
    gn, bn = torch.randn(C, generator=g), torch.randn(C, generator=g)
    tabs = tuple(torch.randn(9, Cout, generator=g) for _ in range(4))
    got = ops.norm2_fold(chan.to(DEV), 1024, gn.to(DEV), bn.to(DEV), tuple(t.to(DEV) for t in tabs))
    ref = E.norm2_fold(chan, 1024, gn, bn, tabs)
    for name, a, r in zip(("mrE", "Ef", "res_scale", "res_shift"), got, ref):
        _close(f"norm2_fold {name}", a, r, rtol=1e-4, atol=1e-4)
    # conv epilogues with a per-frame table and an affine residual
    try:
        for (H, W, Cin, Cout, F_, modes) in [(16, 16, 128, 256, 3, ((1, 1), (0x101, 1), (0, 1))), (32, 32, 128, 128, 2, ((1, 1), (1, 5), (1, 0))), (64, 64, 128, 128, 3, ((1, 1), (1, 5))),
                                             (8, 8, 64, 64, 5, ((1, 1),))]:
            x = E.to_zp(_rand((F_, H, W, Cin), g))
            Wb = _rand((Cout, 9 * Cin), g, (9 * Cin) ** -0.5)
            mrE = torch.stack([torch.zeros(F_), torch.rand(F_, generator=g) + 0.5], 1)
            Ef = torch.randn(F_, 9, Cout, generator=g)
            res = E.to_zp(_rand((F_, H, W, Cout), g))
            rs, rb = torch.randn(F_, Cout, generator=g), torch.randn(F_, Cout, generator=g)
            mr = torch.stack([torch.randn(F_, generator=g) * 0.3, torch.rand(F_, generator=g) + 0.5], 1)
            S1, S2 = torch.randn(9, Cout, generator=g), torch.randn(9, Cout, generator=g)
            for pair, swap in modes:
                nat.lib().vpt_set_conv_pair_mode(pair)
                nat.lib().vpt_set_conv_swap_mode(swap)
                got, gmr = ops.conv3x3_zp(x.to(DEV), Wb.to(DEV), H, W, mr=mrE.to(DEV), Ef=Ef.to(DEV), relu=1)
                ref, rmr = E.conv3x3_zp(x, Wb, H, W, mr=mrE, Ef=Ef, relu=1)
                nat.device_check()
                _close(f"conv Ef pair={pair:#x} swap={swap} {Cin}->{Cout}@{H}", got, ref)
                _close("conv Ef stats", gmr, rmr, rtol=2e-3, atol=2e-3, l2=1e-3)
                got, gmr = ops.conv3x3_zp(x.to(DEV), Wb.to(DEV), H, W, mr=mr.to(DEV), S1=S1.to(DEV), S2=S2.to(DEV), relu=1, residual=res.to(DEV),
                                          res_scale=rs.to(DEV), res_shift=rb.to(DEV))
                ref, rmr = E.conv3x3_zp(x, Wb, H, W, mr=mr, S1=S1, S2=S2, relu=1, residual=res, res_scale=rs, res_shift=rb)
                nat.device_check()
                _close(f"conv affine residual pair={pair:#x} swap={swap} {Cin}->{Cout}@{H}", got, ref)
                gc = got.cpu()
                assert (gc[:, -1] == 0).all() and (gc[:, :, -1] == 0).all()
    finally:
        nat.lib().vpt_set_conv_pair_mode(1)
        nat.lib().vpt_set_conv_swap_mode(1)
