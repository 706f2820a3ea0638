"""GPU: vpt_conv3x3_zp where the epilogue's row map decides what is written.  An epilogue warp finishes the rows its own wgmma
fragment holds: rows 16w .. 16w+15 of each 64-row half of a tile, so a warp's 32 rows are two separate runs.  The cases here end the
last tile inside a first-half run (Q mod 128 = 8), inside a second-half run (72) and eight rows short of a full tile (120), with
Cout = 128 (128-column tiles, four full chunks) and Cout = 64, for the plain, residual, Ef and affine-residual epilogues: output and
statistics against the torch emulation, the ZP zero row / column still written as zeros, and nothing written past the last row."""
import pytest
import torch

import emu_ops as E
import vpt_b200  # noqa: F401
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = 12345.0


def _close(name, got, ref, rtol=2e-2, atol=2e-2, l2=4e-3):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = (got - ref).abs()
    rel = (got - ref).norm() / ref.norm().clamp(min=1e-20)
    bad = err > atol + rtol * ref.abs()
    assert torch.isfinite(got).all() and not bad.any() and rel < l2, f"{name}: {int(bad.sum())} elements out of tolerance, rel l2 {rel:.3g}"


@pytest.mark.parametrize("Cout", [128, 64])
# 8 x 8 frames are 81 ZP rows each; from 64 row tiles on (the last three) Cout = 128 runs as 128-column tiles
@pytest.mark.parametrize("F_,tail", [(8, 8), (72, 72), (120, 120), (136, 8), (200, 72)])
def test_conv3x3_zp_rowmap(F_, tail, Cout):
    H = W = 8
    Cin = 64
    assert (F_ * (H + 1) * (W + 1)) % 128 == tail
    g = torch.Generator().manual_seed(11)
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
        ("affine residual", dict(mr=mr, S1=S1, S2=S2, residual=res, res_scale=rs, res_shift=rb)),
    ]
    for name, kw in cases:
        # the output is the head of a larger buffer: the frame after it must keep its fill
        buf = torch.full((F_ + 1, H + 1, W + 1, Cout), SENTINEL, dtype=torch.bfloat16, device=DEV)
        got, gmr = ops.conv3x3_zp(d(x), d(Wb), H, W, relu=1, out=buf[:F_], **{k: d(v) for k, v in kw.items()})
        nat.device_check()
        ref, rmr = E.conv3x3_zp(x, Wb, H, W, relu=1, **kw)
        assert (buf[F_] == SENTINEL).all(), f"{name}: rows past the last one were written"
        gc = got.cpu()
        assert (gc[:, -1] == 0).all() and (gc[:, :, -1] == 0).all(), f"{name}: ZP zero row / column not maintained"
        _close(f"conv3x3_zp {name} {F_}x{H}x{W} {Cin}->{Cout}", got, ref)
        _close(f"conv3x3_zp {name} stats", gmr, rmr, rtol=2e-3, atol=2e-3, l2=1e-3)
