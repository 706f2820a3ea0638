"""`augment_frames` on the H100: the kernel (`vpt_augment_frames`) against a float64 restatement of its six steps on the same fp32 matrices,
identity and integer-shift exactness, per-sequence broadcast, batch-slice and rerun bit-identity, fully overwritten 0xFF / NaN outputs,
the shared-memory refusal, and the BC and IDM trainers on identity-augmented frames equal to the un-augmented call bit for bit.
tests/test_augment.py checks the host side on the CPU."""
import pytest
import torch

import vpt_b200
from common import make_policy, small_kwargs
from test_idm_training import make_batch, make_idm
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.agent import augment_frames, augment_params, augment_rows
from video_pre_training_b200.training import BCTrainer, IDMTrainer

pytestmark = pytest.mark.gpu

SIZES = [(128, 128), (96, 160), (17, 23)]  # (H, W); 17 x 23 x 3 bytes is no multiple of 16: the staging's tail path
WIDE = dict(rotate=40.0, scale=(0.6, 1.6), shear=25.0, translate=30.0, brightness=(0.4, 1.8), contrast=(0.3, 1.8), saturation=(0.0, 2.0),
            hue=0.5)
IDENT = torch.tensor([0, 1, 0, 0, 0, 1, 1, 1, 0], dtype=torch.float32)


def _grey(p):
    return 0.299 * p[..., 0] + 0.587 * p[..., 1] + 0.114 * p[..., 2]


def _hue64(p, h):
    """torchvision's _rgb2hsv / hue shift / _hsv2rgb in float64 on the [0, 1] scale, back on the uint8 scale."""
    x = p / 255.0
    r, g, b = x.unbind(-1)
    maxc, minc = x.max(-1).values, x.min(-1).values
    eqc = maxc == minc
    cr = maxc - minc
    one = torch.ones_like(maxc)
    s = cr / torch.where(eqc, one, maxc)
    crd = torch.where(eqc, one, cr)
    rc, gc, bc = (maxc - r) / crd, (maxc - g) / crd, (maxc - b) / crd
    hr = (maxc == r) * (bc - gc)
    hg = ((maxc == g) & (maxc != r)) * (2.0 + rc - bc)
    hb = ((maxc != g) & (maxc != r)) * (4.0 + gc - rc)
    hh = torch.fmod((hr + hg + hb) / 6.0 + 1.0, 1.0)
    hh = torch.remainder(hh + h, 1.0)
    v = maxc
    i = torch.floor(hh * 6.0)
    f = hh * 6.0 - i
    i = i.to(torch.int64) % 6
    pp = (v * (1.0 - s)).clamp(0, 1)
    q = (v * (1.0 - s * f)).clamp(0, 1)
    t = (v * (1.0 - s * (1.0 - f))).clamp(0, 1)
    table = torch.stack([torch.stack(c, -1) for c in ((v, t, pp), (q, v, pp), (pp, v, t), (pp, q, v), (t, pp, v), (v, pp, q))], -2)
    out = torch.gather(table, -2, i[..., None, None].expand(*i.shape, 1, 3)).squeeze(-2)
    return (out * 255.0).clamp(0, 255)


def reference(frames, rows):
    """float64 restatement of the kernel's steps 1-5 on the fp32 rows it receives: u8 (N, H, W, 3), rows (N, 10) -> float64 (N, H, W, 3)."""
    N, H, W, _ = frames.shape
    src = frames.double()
    r = rows.double()
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=frames.device),
                            torch.arange(W, dtype=torch.float64, device=frames.device), indexing="ij")
    A = r[:, :6].view(N, 2, 3)[:, :, :, None, None]
    u = (A[:, 0, 0] * xs + A[:, 0, 1] * ys + A[:, 0, 2]).clamp(-2, W + 1)
    v = (A[:, 1, 0] * xs + A[:, 1, 1] * ys + A[:, 1, 2]).clamp(-2, H + 1)
    u0, v0 = torch.floor(u), torch.floor(v)
    fx, fy = (u - u0)[..., None], (v - v0)[..., None]
    x0, y0 = u0.long(), v0.long()
    n = torch.arange(N, device=frames.device)[:, None, None]

    def tap(yy, xx):
        inside = ((xx >= 0) & (xx < W) & (yy >= 0) & (yy < H))[..., None]
        return src[n, yy.clamp(0, H - 1), xx.clamp(0, W - 1)] * inside

    p00, p01, p10, p11 = tap(y0, x0), tap(y0, x0 + 1), tap(y0 + 1, x0), tap(y0 + 1, x0 + 1)
    top, bot = p00 + fx * (p01 - p00), p10 + fx * (p11 - p10)
    p = top + fy * (bot - top)
    b, c, s, h = (r[:, 6 + k, None, None, None] for k in range(4))
    p = torch.where(b != 1, (b * p).clamp(0, 255), p)
    m = _grey(p).mean(dim=(1, 2))[:, None, None, None]
    p = torch.where(c != 1, (c * p + (1 - c) * m).clamp(0, 255), p)
    p = torch.where(s != 1, (s * p + (1 - s) * _grey(p)[..., None]).clamp(0, 255), p)
    return torch.where(h != 0, _hue64(p, h[..., 0]), p).clamp(0, 255)


def _rows(params, shape):
    return torch.from_numpy(augment_rows(params, shape)).cuda()


def _frames(g, N, H, W):
    return torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g).cuda()


def _wide_params(g, N):
    """WIDE draws, with every colour factor at its identity in about a third of the frames (the kernel skips those steps)."""
    p = augment_params(N, generator=g, **WIDE)
    keep = torch.rand((N, 4), generator=g) < 0.35
    p[:, 5:9] = torch.where(keep, IDENT[5:9], p[:, 5:9])
    return p


@pytest.mark.parametrize("H,W", SIZES)
def test_matches_float64(H, W):
    g = torch.Generator().manual_seed(H * 1000 + W)
    N = 24
    frames = _frames(g, N, H, W)
    p = _wide_params(g, N)
    ref = reference(frames, _rows(p, frames.shape))
    got32 = augment_frames(frames, p, out_dtype=torch.float32)
    got8 = augment_frames(frames, p)
    torch.cuda.synchronize()
    nat.device_check()
    err = (got32.double() - ref).abs().max().item()
    print(f"{H}x{W}: fp32 max abs err {err:.2e}")
    assert err < 2e-3, err
    near = ((ref - torch.floor(ref)) - 0.5).abs() < 1e-3  # within 1e-3 of a rounding boundary: either neighbour is right
    rounded = torch.round(ref).to(torch.uint8)  # half to even
    bad = (got8 != rounded) & ~near
    print(f"{H}x{W}: u8 mismatches outside the boundary band {int(bad.sum())}, in it {int(((got8 != rounded) & near).sum())}")
    assert not bad.any()
    assert ((got8.double() - ref).abs() <= 0.5 + 1e-3).all()
    # the output is not trivially the input: the random warps and colours moved most pixels
    assert (got8 != frames).float().mean() > 0.5


@pytest.mark.parametrize("H,W", SIZES)
def test_identity_is_exact(H, W):
    g = torch.Generator().manual_seed(7)
    frames = _frames(g, 5, H, W)
    ident = IDENT.repeat(5, 1)
    assert torch.equal(augment_frames(frames, ident), frames)
    assert torch.equal(augment_frames(frames, ident, out_dtype=torch.float32), frames.float())
    # a frame base that is not 16-byte aligned takes the byte-wise staging
    buf = torch.empty(5 * H * W * 3 + 1, dtype=torch.uint8, device="cuda")
    odd = buf[1:].view(5, H, W, 3)
    odd.copy_(frames)
    assert odd.data_ptr() % 16 != 0
    assert torch.equal(augment_frames(odd, ident), frames)
    p = _wide_params(g, 5)
    assert torch.equal(augment_frames(odd, p), augment_frames(frames, p))


@pytest.mark.parametrize("H,W", SIZES)
def test_integer_translation_is_a_shift(H, W):
    g = torch.Generator().manual_seed(8)
    frames = _frames(g, 4, H, W)
    shifts = [(5, -3), (-7, 2), (0, 9), (W + 1, 0)]
    p = IDENT.repeat(4, 1)
    for i, (tx, ty) in enumerate(shifts):
        p[i, 3], p[i, 4] = tx, ty
    for dt in (torch.uint8, torch.float32):
        out = augment_frames(frames, p, out_dtype=dt)
        for i, (tx, ty) in enumerate(shifts):
            want = torch.zeros_like(frames[i])
            ys, xs = slice(max(ty, 0), min(H + ty, H)), slice(max(tx, 0), min(W + tx, W))
            if ys.start < ys.stop and xs.start < xs.stop:
                want[ys, xs] = frames[i, max(-ty, 0):max(-ty, 0) + ys.stop - ys.start, max(-tx, 0):max(-tx, 0) + xs.stop - xs.start]
            assert torch.equal(out[i], want.to(dt)), (dt, tx, ty)


def test_per_sequence_params_broadcast():
    g = torch.Generator().manual_seed(9)
    B, T, H, W = 3, 6, 128, 128
    seq = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g).cuda()
    p = augment_params(B, generator=g, **WIDE)
    out = augment_frames(seq, p)
    assert out.shape == seq.shape and out.dtype == torch.uint8
    assert torch.equal(out, augment_frames(seq, p[:, None].expand(B, T, 9).contiguous()))
    assert torch.equal(out.view(B * T, H, W, 3), augment_frames(seq.view(B * T, H, W, 3), p.repeat_interleave(T, 0)))
    # the same warp on every frame of a sequence: a sequence of one repeated frame gives one repeated output, and each frame equals
    # that frame augmented alone with its sequence's row
    rep = seq[:, :1].expand(B, T, H, W, 3).contiguous()
    o = augment_frames(rep, p, out_dtype=torch.float32)
    assert all(torch.equal(o[b, t], o[b, 0]) for b in range(B) for t in range(T))
    for b in range(B):
        for t in (0, T - 1):
            assert torch.equal(out[b, t], augment_frames(seq[b, t][None], p[b][None])[0])
    per_frame = augment_params(B, T, generator=g, per_frame=True, **WIDE)
    assert torch.equal(augment_frames(seq, per_frame)[1, 2], augment_frames(seq[1, 2][None], per_frame[1, 2][None])[0])


@pytest.mark.parametrize("dt", [torch.uint8, torch.float32])
def test_slices_reruns_and_prefilled_outputs(dt):
    g = torch.Generator().manual_seed(10)
    N, H, W = 40, 128, 128
    frames = _frames(g, N, H, W)
    p = _wide_params(g, N)
    whole = augment_frames(frames, p, out_dtype=dt)
    for lo, hi in ((0, 1), (3, 7), (17, 40), (39, 40)):
        assert torch.equal(augment_frames(frames[lo:hi], p[lo:hi], out_dtype=dt), whole[lo:hi]), (lo, hi)
    for _ in range(2):
        assert torch.equal(augment_frames(frames, p, out_dtype=dt), whole)
    rows = _rows(p, frames.shape)
    fills = [lambda o: o.view(torch.uint8).fill_(0xFF)] + ([lambda o: o.fill_(float("nan"))] if dt == torch.float32 else [])
    for fill in fills:
        out = torch.empty((N, H, W, 3), dtype=dt, device="cuda")
        fill(out)
        ops.augment(frames, rows, out)
        torch.cuda.synchronize()
        assert torch.equal(out, whole)


def test_refuses_a_frame_larger_than_shared_memory():
    cap = nat.lib().vpt_augment_max_frame_bytes()
    print("largest frame:", cap, "bytes")
    assert cap >= 128 * 128 * 3
    W = cap // (3 * 64) + 1  # 64 x W x 3 > cap
    big = torch.zeros((2, 64, W, 3), dtype=torch.uint8, device="cuda")
    n0 = ops.LAUNCHES
    with pytest.raises(nat.NativeError, match="shared memory"):
        augment_frames(big, IDENT.repeat(2, 1))
    assert ops.LAUNCHES == n0
    fits = torch.randint(0, 256, (2, 64, cap // (3 * 64), 3), dtype=torch.uint8, device="cuda")
    assert torch.equal(augment_frames(fits, IDENT.repeat(2, 1)), fits)


def _step(tr, mod, img, first, actions):
    for p in mod.parameters():
        p.grad = None
    loss, _ = tr.loss_and_grad(img, first, mod.initial_state(img.shape[0]), actions)
    torch.cuda.synchronize()
    nat.device_check()
    grads = {}
    for n, p in mod.named_parameters():
        grads[n], p.grad = p.grad, None
    return loss, grads


def _same(a, b):
    (la, ga), (lb, gb) = a, b
    assert torch.equal(la, lb)
    assert ga.keys() == gb.keys()
    for n in ga:
        assert (ga[n] is None) == (gb[n] is None), n
        assert ga[n] is None or torch.equal(ga[n], gb[n]), n


def test_trainers_on_identity_augmentation_bit_identical():
    g = torch.Generator().manual_seed(11)
    pol, _, _ = make_policy(small_kwargs())
    pol = pol.cuda()
    B, T = 2, 8
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    tr = BCTrainer(pol)
    ident = augment_params(B, generator=g)
    base = _step(tr, pol, img, first, actions)
    _same(_step(tr, pol, augment_frames(img, ident), first, actions), base)
    f32 = augment_frames(img, ident, out_dtype=torch.float32)
    assert f32.dtype == torch.float32
    _same(_step(tr, pol, f32, first, actions), base)

    idm, _, _ = make_idm()
    idm = idm.cuda()
    img, first, actions = make_batch(g)
    img, first, actions = img.cuda(), first.cuda(), {k: v.cuda() for k, v in actions.items()}
    tr = IDMTrainer(idm)
    ident = augment_params(img.shape[0], generator=g)
    base = _step(tr, idm, img, first, actions)
    _same(_step(tr, idm, augment_frames(img, ident), first, actions), base)
    _same(_step(tr, idm, augment_frames(img, ident, out_dtype=torch.float32), first, actions), base)
    # a real augmentation changes the loss (the frames reach the model)
    aug = augment_frames(img, augment_params(img.shape[0], generator=g, **WIDE))
    assert not torch.equal(_step(tr, idm, aug, first, actions)[0], base[0])
    assert vpt_b200.augment_frames is augment_frames
