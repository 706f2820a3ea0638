"""GPU: vpt_conv3x3_zp at shapes that exercise the tile schedule and the epilogue paths of the ping-pong kernel rather than the
layer shapes of the model: a CTA with a single tile (the second MMA warpgroup has none), CTAs with an odd number of tiles,
a CTA count that leaves some CTAs one tile more than others, and Cout values whose last 32-column chunk is partial (the
element-by-element epilogue path) next to full chunks (the coalesced path).  Each case runs the plain, residual, Ef and affine-residual
epilogues against the torch emulation."""
import pytest
import torch

import emu_ops as E
import vpt_b200  # noqa: F401
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _close(name, got, ref, rtol=2e-2, atol=2e-2, l2=4e-3):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = (got - ref).abs()
    rel = (got - ref).norm() / ref.norm().clamp(min=1e-20)
    bad = err > atol + rtol * ref.abs()
    assert torch.isfinite(got).all() and not bad.any() and rel < l2, f"{name}: {int(bad.sum())} elements out of tolerance, rel l2 {rel:.3g}"


@pytest.mark.parametrize("H,W,Cin,Cout,F_", [
    (8, 8, 64, 16, 1),      # one 128-row tile: a single CTA whose second warpgroup has no tile; Cout 16 = one partial chunk
    (8, 8, 64, 48, 1),      # a full 32-column chunk and a partial one in the same tile
    (8, 8, 128, 80, 3),     # few tiles: 64-column tiles, the second one a partial chunk only; two channel blocks
    (8, 8, 64, 64, 209),    # 133 row tiles: on 132 SMs one CTA runs two tiles, the others one
    (16, 16, 128, 128, 175),  # 396 row tiles: three per CTA on 132 SMs (odd count: warpgroup 0 runs two, warpgroup 1 one)
    (16, 16, 256, 256, 29),   # two column tiles per row tile, four channel blocks per tile
])
def test_conv3x3_zp_schedule(H, W, Cin, Cout, F_):
    g = torch.Generator().manual_seed(7)
    x = E.to_zp((torch.randn(F_, H, W, Cin, generator=g)).to(torch.bfloat16))
    Wb = (torch.randn(Cout, 9 * Cin, generator=g) * (9 * Cin) ** -0.5).to(torch.bfloat16)
    mr = torch.stack([torch.randn(F_, generator=g) * 0.3, torch.rand(F_, generator=g) + 0.5], 1)
    mrE = torch.stack([torch.zeros(F_), torch.rand(F_, generator=g) + 0.5], 1)
    S1, S2 = torch.randn(9, Cout, generator=g), torch.randn(9, Cout, generator=g)
    Ef = torch.randn(F_, 9, Cout, generator=g)
    res = E.to_zp(torch.randn(F_, H, W, Cout, generator=g).to(torch.bfloat16))
    rs, rb = torch.randn(F_, Cout, generator=g), torch.randn(F_, Cout, generator=g)
    d = lambda t: t.to(DEV)  # noqa: E731
    cases = [
        ("plain", dict(mr=mr, S1=S1, S2=S2)),
        ("residual", dict(mr=mr, S1=S1, S2=S2, residual=res)),
        ("Ef", dict(mr=mrE, Ef=Ef)),
    ]
    if Cout % 8 == 0:
        cases.append(("affine residual", dict(mr=mr, S1=S1, S2=S2, residual=res, res_scale=rs, res_shift=rb)))
    for name, kw in cases:
        got, gmr = ops.conv3x3_zp(d(x), d(Wb), H, W, relu=1, **{k: d(v) for k, v in kw.items()})
        nat.device_check()
        ref, rmr = E.conv3x3_zp(x, Wb, H, W, relu=1, **kw)
        gc = got.cpu()
        assert (gc[:, -1] == 0).all() and (gc[:, :, -1] == 0).all(), f"{name}: ZP zero row / column not maintained"
        _close(f"conv3x3_zp {name} {F_}x{H}x{W} {Cin}->{Cout}", got, ref)
        _close(f"conv3x3_zp {name} stats", gmr, rmr, rtol=2e-3, atol=2e-3, l2=1e-3)
    # dgrad form: no fold, no ReLU, no statistics
    got, _ = ops.conv3x3_zp(d(x), d(Wb), H, W, relu=0, want_stats=False)
    nat.device_check()
    ref, _ = E.conv3x3_zp(x, Wb, H, W, relu=0, want_stats=False)
    _close(f"conv3x3_zp dgrad {F_}x{H}x{W} {Cin}->{Cout}", got, ref)
