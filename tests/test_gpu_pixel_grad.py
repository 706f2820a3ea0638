"""Float frames and the image gradient on the H100: the two image-gradient kernels against the float64 closed forms of
tests/pixel_refs.py at the released shapes, the first conv's two backward kernels against each other, the fp32-frame forward kernels
bit-identical to uint8 on integer frames, and `loss.backward()` to the pixels at 2x, checked against the same call's first-conv weight
gradient and against the all-frozen call.  tests/test_pixel_grad.py
checks the host logic on the CPU."""
import copy
import gc

import pytest
import torch

import emu_autograd_ops
import emu_idm_ops
import emu_ops
import emu_pixel_ops
import pixel_refs
import vpt_b200
from common import perturb
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops

pytestmark = pytest.mark.gpu

PAD = 256  # fp32 NaN guard elements before and after each image-gradient buffer


@pytest.fixture(autouse=True)
def _free_device_memory():
    """A differentiable policy and its autograd runner reference each other: collect them after each test, so that the 2x / 4x
    policies made here do not hold device memory into the tests that run after this file."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300)).item()


def _frames(g, F_, f32, H=128, W=128):
    if f32:
        return (torch.rand((F_, H, W, 3), generator=g) * 340.0 - 40.0).cuda()  # non-integer, outside [0, 255]
    return torch.randint(0, 256, (F_, H, W, 3), dtype=torch.uint8, generator=g).cuda()


def _weights(g, C0):
    w = (torch.randn((C0, 27), generator=g) * 0.2 / 255.0).cuda()
    b = (torch.randn((C0,), generator=g) * 0.05).cuda()
    return w, b


def _dy(g, F_, Ho, Wo, C):
    dy = torch.randn((F_, Ho + 1, Wo + 1, C), generator=g).to(torch.bfloat16)
    dy[:, -1] = 0
    dy[:, :, -1] = 0
    return dy.cuda()


def _guarded(n):
    buf = torch.full((n + 2 * PAD,), float("nan"), device="cuda")
    return buf, buf[PAD:PAD + n]


def _fc_dimg(img, w, b, dy, C0):
    F_, H, W, _ = img.shape
    buf, out = _guarded(F_ * H * W * 3)
    nat.check(nat.lib().vpt_firstconv_dimg(img.data_ptr(), int(img.dtype == torch.float32), w.data_ptr(), b.data_ptr(), dy.data_ptr(), out.data_ptr(),
                                           F_, H, W, C0, None), "vpt_firstconv_dimg")
    torch.cuda.synchronize()
    assert torch.isnan(buf[:PAD]).all() and torch.isnan(buf[-PAD:]).all(), "guard band written"
    return out.view(F_, H, W, 3).clone()


@pytest.mark.parametrize("C0", [64, 128, 192, 256])
@pytest.mark.parametrize("f32", [False, True])
def test_firstconv_dimg_matches_float64(C0, f32):
    g = torch.Generator().manual_seed(C0 + f32)
    F_ = 3
    img, (w, b), dy = _frames(g, F_, f32), _weights(g, C0), _dy(g, F_, 64, 64, C0)
    out = _fc_dimg(img, w, b, dy, C0)
    assert torch.isfinite(out).all()
    ref = pixel_refs.firstconv_dimg(img, w, b, dy, C0)
    err = _rel(out, ref)
    print(f"firstconv_dimg C0={C0} f32={f32}: rel L2 {err:.2e}")
    assert err < 2e-3
    assert torch.equal(out, _fc_dimg(img, w, b, dy, C0)), "not bit-reproducible"


@pytest.mark.parametrize("f32", [False, True])
def test_first_conv_backward_kernels_agree(f32):
    """With the routing fixed, sum dimg * x and sum dW * w (+ db * b) both equal sum dpre * (w * x + b): the two kernels differentiate one
    function."""
    g = torch.Generator().manual_seed(7 + f32)
    C0, F_ = 128, 5
    img, (w, b), dy = _frames(g, F_, f32), _weights(g, C0), _dy(g, F_, 64, 64, C0)
    dimg = _fc_dimg(img, w, b, dy, C0)
    dW, db = ops.firstconv_bwd(img, w, b, dy, C0)
    x, dpre = pixel_refs.routed(img, w, b, dy, C0)
    pre = torch.nn.functional.conv2d(x, w.double().reshape(C0, 3, 3, 3).permute(0, 3, 1, 2), padding=1)
    s_ref = (dpre * pre).sum().item()
    s_img = (dimg.double() * img.double()).sum().item()
    s_w = (dW.double() * w.double()).sum().item()
    print(f"sum dpre*(w*x) {s_ref:.6e}, sum dimg*x {s_img:.6e}, sum dW*w {s_w:.6e}")
    assert abs(s_img - s_ref) < 1e-3 * abs(s_ref) and abs(s_w - s_ref) < 1e-3 * abs(s_ref)


def _c3_dimg(dy, w, B, T, H, W):
    buf, out = _guarded(B * T * H * W * 3)
    nat.check(nat.lib().vpt_conv3d_t5_dimg(dy.data_ptr(), w.data_ptr(), out.data_ptr(), B, T, H, W, w.shape[0], None), "vpt_conv3d_t5_dimg")
    torch.cuda.synchronize()
    assert torch.isnan(buf[:PAD]).all() and torch.isnan(buf[-PAD:]).all(), "guard band written"
    return out.view(B * T, H, W, 3).clone()


@pytest.mark.parametrize("B,T", [(3, 1), (3, 37), (1, 128)])
def test_conv3d_t5_dimg_matches_float64(B, T):
    g = torch.Generator().manual_seed(B * 1000 + T)
    C, H, W = 128, 128, 128
    w = (torch.randn((C, 15), generator=g) / 255.0).cuda()
    dy = _dy(g, B * T, H, W, C)
    out = _c3_dimg(dy, w, B, T, H, W)
    ref = pixel_refs.conv3d_t5_dimg(dy, w, B, T, H, W)
    err = _rel(out, ref)
    print(f"conv3d_t5_dimg B={B} T={T}: rel L2 {err:.2e}, max abs {(out.double() - ref).abs().max().item():.2e}")
    assert err < 1e-5
    assert torch.equal(out, _c3_dimg(dy, w, B, T, H, W)), "not bit-reproducible"


def _agent(width):
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    return pol.cuda()


def test_float_frames_forward_bit_identical_2x():
    """2x at B x T = 16 x 128: fp32 frames holding the uint8 values give pd, vpred and state_out bit for bit, in both precisions, and the
    first-conv kernel alone gives the same outputs and statistics partials."""
    pol = _agent("2x")
    g = torch.Generator().manual_seed(1)
    img = torch.randint(0, 256, (16, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(16, 128, dtype=torch.bool).cuda()
    st = pol.initial_state(16)
    for precision in ("bf16", "fp32"):
        pol.set_precision(precision)
        with torch.no_grad():
            (pd0, v0, _), s0 = pol({"img": img}, first, st)
            (pd1, v1, _), s1 = pol({"img": img.float()}, first, st)
        assert torch.equal(v0, v1) and all(torch.equal(pd0[k], pd1[k]) for k in pd0), precision
        for (_, (k0, w0)), (_, (k1, w1)) in zip(s0, s1):
            assert torch.equal(k0, k1) and torch.equal(w0, w1)
    pol.set_precision("bf16")
    st0 = pol.net.prepared().stacks[0]
    frames = img.view(-1, 128, 128, 3)[:2048]
    C0 = pol.net.cfg.chans[0]
    for zp in (True, False):
        a = ops.firstconv_pool(frames, st0["fc_w"], st0["fc_b"], C0, zp=zp, want_chan=True)
        b = ops.firstconv_pool(frames.float(), st0["fc_w"], st0["fc_b"], C0, zp=zp, want_chan=True)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_float_frames_forward_bit_identical_4x_idm():
    torch.manual_seed(0)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()
    g = torch.Generator().manual_seed(2)
    img = torch.randint(0, 256, (2, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(2, 128, dtype=torch.bool).cuda()
    with torch.no_grad():
        (pd0, _, _), _ = pol({"img": img}, first, pol.initial_state(2))
        (pd1, _, _), _ = pol({"img": img.float()}, first, pol.initial_state(2))
    assert all(torch.equal(pd0[k], pd1[k]) for k in pd0)
    prep = pol.net.prepared()
    a = ops.conv3d_t5(img, prep.conv3d[0], prep.conv3d[1], pol.net.cfg.conv3d_out)
    b = ops.conv3d_t5(img.float(), prep.conv3d[0], prep.conv3d[1], pol.net.cfg.conv3d_out)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _camera_loss(pd):
    return -pd["camera"][..., 0, :7].sum() / pd["camera"].numel()


def test_loss_backward_to_the_pixels_2x():
    """2x, B = 2, T = 16 non-integer frames, the camera-head loss.  All trainable: img.grad and the first conv's weight gradient come from
    the same routed pre-pool gradient dpre, so sum img.grad * img == sum dW * W (both are sum dpre * (W/255 * img)) up to fp32 rounding.
    All frozen: img.grad is the all-trainable call's bit for bit, and no parameter gets a gradient."""
    pol = _agent("2x").set_autograd(True)
    g = torch.Generator().manual_seed(3)
    img = (torch.rand((2, 16, 128, 128, 3), generator=g) * 340.0 - 40.0).cuda()
    first = torch.zeros(2, 16, dtype=torch.bool).cuda()
    x = img.clone().requires_grad_(True)
    (pd, _, _), _ = pol({"img": x}, first, pol.initial_state(2))
    _camera_loss(pd).backward()
    nat.device_check()
    assert torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0
    wt = dict(pol.named_parameters())["net.img_process.cnn.stacks.0.firstconv.layer.weight"]
    s_img = (x.grad.double() * img.double()).sum().item()
    s_w = (wt.grad.double() * wt.detach().double()).sum().item()
    print(f"2x: sum img.grad * img {s_img:.6e}, sum dW * W {s_w:.6e}")
    assert abs(s_img - s_w) < 1e-3 * abs(s_w)
    for p in pol.parameters():
        p.requires_grad_(False)
        p.grad = None
    y = img.clone().requires_grad_(True)
    (pd, _, _), _ = pol({"img": y}, first, pol.initial_state(2))
    _camera_loss(pd).backward()
    assert torch.equal(y.grad, x.grad)
    assert all(p.grad is None for p in pol.parameters())


def _grad_on(fn, *a, **k):
    with torch.enable_grad():
        return fn(*a, **k)


def _emulated_img_grad(mod, img, first, loss_fn, exact):
    """The same `loss.backward()` to the pixels on the CPU through the test-only emulation of every op (the two image-gradient ops
    included): bf16 rounding where the kernels round (exact=False), or fp32 everywhere (exact=True, the function the kernels approximate)."""
    from video_pre_training_b200 import policy, training

    mp = pytest.MonkeyPatch()
    try:
        for m in (emu_ops, emu_idm_ops, emu_autograd_ops):
            for name in dir(m):
                if not name.startswith("_") and callable(getattr(m, name)) and hasattr(ops, name):
                    mp.setattr(ops, name, getattr(m, name))
        for name in ("firstconv_bwd", "maxpool3s2_bwd", "attention_bwd"):
            mp.setattr(ops, name, lambda *a, _fn=getattr(emu_ops, name), **k: _grad_on(_fn, *a, **k))
        mp.setattr(ops, "conv3d_t5_bwd", lambda *a, **k: _grad_on(emu_idm_ops.conv3d_t5_bwd, *a, **k))
        mp.setattr(ops, "firstconv_dimg", lambda *a, **k: _grad_on(emu_pixel_ops.firstconv_dimg, *a, **k))
        mp.setattr(ops, "conv3d_t5_dimg", emu_pixel_ops.conv3d_t5_dimg)
        if exact:
            for m in (emu_ops, policy, training):
                mp.setattr(m, "BF16", torch.float32)
        x = img.detach().cpu().clone().requires_grad_(True)
        (pd, _, _), _ = mod({"img": x}, first.cpu(), mod.initial_state(img.shape[0]))
        loss_fn(pd).backward()
        return x.grad
    finally:
        mp.undo()


def _vs_emulation(mod, img, first, loss_fn, what):
    """img.grad of the CUDA step against the emulated CPU step.  The bf16 step is one rounding of the fp32 function; the CUDA kernels round
    at other places (fused epilogues, the conv's tile order), and after a max-pool / ReLU mask flip deep in the net the two roundings take
    different paths back to the pixels.  So the bound is relative to the emulation's own rounding error: the CUDA gradient must be as
    close to the fp32 emulation as the bf16 emulation is (within 2x), and within 5e-2 when that error is smaller."""
    x = img.clone().requires_grad_(True)
    (pd, _, _), _ = mod({"img": x}, first, mod.initial_state(img.shape[0]))
    loss_fn(pd).backward()
    nat.device_check()
    got = x.grad.cpu()
    assert torch.isfinite(got).all() and got.abs().sum() > 0
    bf16 = _emulated_img_grad(copy.deepcopy(mod).cpu(), img, first, loss_fn, exact=False)
    f32 = _emulated_img_grad(copy.deepcopy(mod).cpu(), img, first, loss_fn, exact=True)
    e_gpu, e_emu, e_pair = _rel(got, f32), _rel(bf16, f32), _rel(got, bf16)
    print(f"{what}: img.grad rel L2, CUDA vs fp32 emulation {e_gpu:.2e}, bf16 emulation vs fp32 {e_emu:.2e}, CUDA vs bf16 emulation {e_pair:.2e}")
    assert e_gpu < max(5e-2, 2 * e_emu)


def test_loss_backward_to_the_pixels_2x_matches_emulation():
    """2x, every parameter frozen, B = 1, T = 8 non-integer frames, the camera-head loss."""
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
    pol.requires_grad_(False)
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(4)
    img = (torch.rand((1, 8, 128, 128, 3), generator=g) * 340.0 - 40.0).cuda()
    _vs_emulation(pol, img, torch.zeros(1, 8, dtype=torch.bool).cuda(), _camera_loss, "2x")


def test_idm_loss_backward_to_the_pixels_4x_matches_emulation():
    """The released 4x IDM (T = 2 per sequence), every parameter frozen, B = 2 with recompute_frames = 2: two recomputed chunks, each
    writing its sequence's slice of the image gradient through vpt_conv3d_t5_dimg."""
    torch.manual_seed(0)
    kw = vpt_b200.idm_net_kwargs(timesteps=2, attention_memory_size=2)  # mask "none": memory size == timesteps (no KV memory)
    idm = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), kw).cuda()
    idm.requires_grad_(False)
    idm.set_autograd(True, recompute_frames=2)
    g = torch.Generator().manual_seed(5)
    img = (torch.rand((2, 2, 128, 128, 3), generator=g) * 340.0 - 40.0).cuda()
    _vs_emulation(idm, img, torch.zeros(2, 2, dtype=torch.bool).cuda(), _camera_loss, "4x IDM")
