"""Float frames and the image gradient on the CPU, through the test-only torch emulation of the ops (tests/emu_pixel_ops.py for the two
image-gradient ops): integer-valued float frames give exactly the uint8 results everywhere frames enter, and `loss.backward()` with an
`img` that requires grad writes `img.grad`, the gradient of torch autograd through the emulated forward, while trainable parameters get
exactly the gradients of the same call without it.  tests/test_gpu_pixel_grad.py repeats it through the CUDA kernels."""
import copy

import pytest
import torch

import emu_pixel_ops
import test_rl_training
import vpt_oracle as O
from common import make_policy, small_kwargs
from test_autograd import _with_grad, batch, bc_loss, emulated, exact  # noqa: F401  (fixtures)
from test_freeze import OpLog, freeze
from test_idm_training import make_batch, make_idm
from test_recompute import _grads, assert_same_state, emu  # noqa: F401  (fixture)
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import _autograd_runner
from video_pre_training_b200.training import BCTrainer, IDMTrainer, RLTrainer

IMG_OPS = ("firstconv_dimg", "conv3d_t5_dimg")


@pytest.fixture()
def pix(emu, monkeypatch):  # noqa: F811
    monkeypatch.setattr(ops, "firstconv_dimg", _with_grad(emu_pixel_ops.firstconv_dimg))
    monkeypatch.setattr(ops, "conv3d_t5_dimg", emu_pixel_ops.conv3d_t5_dimg)
    yield


def float_img(g, shape, lo=-40.0, hi=300.0):
    """Non-integer frames with values outside [0, 255]."""
    return torch.rand(shape, generator=g) * (hi - lo) + lo


def freeze_all(mod):
    for p in mod.parameters():
        p.requires_grad_(False)


def camera_loss(pd):
    return -pd["camera"][..., 0, :7].sum() / pd["camera"].numel()


# ---------------------------------------------------------------------------------------------------------------
# integer-valued float frames == uint8 frames, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.float64])
def test_integer_float_frames_equal_uint8_in_inference(pix, dtype):
    pol, _, _ = make_policy(small_kwargs())
    idm, _, _ = make_idm()
    g = torch.Generator().manual_seed(0)
    img, first, _ = batch(g, 2, 8)
    with torch.no_grad():
        for m in (pol, idm):
            (pd0, v0, _), s0 = m({"img": img}, first, m.initial_state(2))
            (pd1, v1, _), s1 = m({"img": img.to(dtype)}, first, m.initial_state(2))
            assert all(torch.equal(pd0[k], pd1[k]) for k in pd0)
            assert (v0 is None and v1 is None) or torch.equal(v0, v1)
            assert_same_state(s0, s1)


def test_integer_float_frames_equal_uint8_in_the_trainers(pix):
    g = torch.Generator().manual_seed(1)
    pol0, _, _ = make_policy(small_kwargs())
    img, first, actions = batch(g, 2, 8)
    res = []
    for im in (img, img.float()):
        pol = copy.deepcopy(pol0)
        loss, st = BCTrainer(pol).loss_and_grad(im, first, pol.initial_state(2), actions)
        res.append((loss, st, _grads(pol)))
    pol0, sd, sd_ref, cfg = test_rl_training.make_pair()
    pd_ref, _ = test_rl_training.ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, 2))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 2))
    old, adv, returns = test_rl_training.make_rl_batch(g, O.logprob(pd0, actions), 2, 8)
    for im in (img, img.double()):
        pol = copy.deepcopy(pol0)
        loss, st = RLTrainer(pol).loss_and_grad(im, first, pol.initial_state(2), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)
        res.append((loss, st, _grads(pol)))
    idm0, _, _ = make_idm()
    img3, first3, actions3 = make_batch(g)
    for im in (img3, img3.half()):
        idm = copy.deepcopy(idm0)
        loss, st = IDMTrainer(idm).loss_and_grad(im, first3, idm.initial_state(2), actions3)
        res.append((loss, st, _grads(idm)))
    for (l0, s0, g0), (l1, s1, g1) in zip(res[0::2], res[1::2]):
        assert torch.equal(l0, l1)
        assert_same_state(s0, s1)
        assert g0.keys() == g1.keys() and all((g0[n] is None) == (g1[n] is None) and (g0[n] is None or torch.equal(g0[n], g1[n])) for n in g0)


@pytest.mark.parametrize("recompute", [None, 8])
def test_integer_float_frames_equal_uint8_in_loss_backward(pix, recompute):
    """The agent (BC loss + value term) and the IDM: pd, state_out and every .grad bit for bit, with and without recompute_frames."""
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(2)
    img, first, actions = batch(g, 2, 8)
    res = []
    for im in (img, img.float()):
        pol = copy.deepcopy(pol0).set_autograd(True, recompute_frames=recompute)
        (pd, vpred, _), st = pol({"img": im}, first, pol.initial_state(2))
        (bc_loss(pol, pd, actions) + 0.1 * (vpred ** 2).mean()).backward()
        res.append((pd, st, _grads(pol)))
    (pd0, s0, g0), (pd1, s1, g1) = res
    assert all(torch.equal(pd0[k], pd1[k]) for k in pd0)
    assert_same_state(s0, s1)
    assert all((g0[n] is None) == (g1[n] is None) and (g0[n] is None or torch.equal(g0[n], g1[n])) for n in g0)
    idm0, _, _ = make_idm()
    img3, first3, actions3 = make_batch(g)
    res = []
    for im in (img3, img3.float()):
        idm = copy.deepcopy(idm0).set_autograd(True, recompute_frames=recompute)
        (pd, _, _), st = idm({"img": im}, first3, idm.initial_state(2))
        (-O.logprob(pd, actions3).mean()).backward()
        res.append((pd, st, _grads(idm)))
    (pd0, s0, g0), (pd1, s1, g1) = res
    assert all(torch.equal(pd0[k], pd1[k]) for k in pd0)
    assert_same_state(s0, s1)
    assert all((g0[n] is None) == (g1[n] is None) and (g0[n] is None or torch.equal(g0[n], g1[n])) for n in g0)


def test_integer_dtypes_still_raise(pix):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(3)
    img, first, _ = batch(g, 1, 2)
    with pytest.raises(TypeError):
        pol({"img": img.to(torch.int32)}, first, pol.initial_state(1))


# ---------------------------------------------------------------------------------------------------------------
# the image gradient
# ---------------------------------------------------------------------------------------------------------------
def oracle_img_grad(sd, cfg, img, first, loss_fn, idm=False, train=False):
    leaf = {k: v.clone().requires_grad_(train and v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}
    x = img.detach().clone().requires_grad_(True)
    fwd = O.idm_policy_forward if idm else O.agent_policy_forward
    (pd, _, _), _ = fwd(leaf, cfg, x, first, O.initial_state(cfg, img.shape[0]))
    loss_fn(pd).backward()
    return x.grad, leaf


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize("recompute", [None, 8])
def test_saliency_all_frozen_is_autograds(pix, exact, recompute):
    """Every parameter frozen: `loss.backward()` writes img.grad only (as float), equal to autograd through the oracle."""
    pol, sd, cfg = make_policy(small_kwargs())
    freeze_all(pol)
    pol.set_autograd(True, recompute_frames=recompute)
    g = torch.Generator().manual_seed(4)
    _, first, _ = batch(g, 2, 8)
    img = float_img(g, (2, 8, 32, 32, 3)).requires_grad_(True)
    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(2))
    camera_loss(pd).backward()
    assert all(p.grad is None for p in pol.parameters())
    ref, _ = oracle_img_grad(sd, cfg, img, first, camera_loss)
    assert img.grad is not None and img.grad.dtype == torch.float32
    assert rel(img.grad, ref) < 5e-2


def test_idm_image_gradient_is_autograds(pix, exact):
    idm, sd, cfg = make_idm()
    freeze_all(idm)
    idm.set_autograd(True, recompute_frames=8)  # B = 2, T = 8: two recomputed chunks, one whole sequence each
    g = torch.Generator().manual_seed(5)
    _, first, actions = make_batch(g)
    img = float_img(g, (2, 8, 32, 32, 3)).requires_grad_(True)
    (pd, _, _), _ = idm({"img": img}, first, idm.initial_state(2))
    loss_fn = lambda p: -O.logprob(p, actions).mean()  # noqa: E731
    loss_fn(pd).backward()
    ref, _ = oracle_img_grad(sd, cfg, img, first, loss_fn, idm=True)
    assert rel(img.grad, ref) < 5e-2


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
def test_leaf_dtype_gets_its_gradient_in_its_own_dtype(pix, exact, dtype):
    pol, sd, cfg = make_policy(small_kwargs())
    freeze_all(pol)
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(6)
    _, first, _ = batch(g, 1, 4)
    img = float_img(g, (1, 4, 32, 32, 3)).to(dtype).requires_grad_(True)
    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(1))
    camera_loss(pd).backward()
    assert img.grad.dtype == dtype
    ref, _ = oracle_img_grad(sd, cfg, img.float(), first, camera_loss)
    assert rel(img.grad.float(), ref) < 5e-2


@pytest.mark.parametrize("pattern", ["all", "cnn", "heads_only"])
def test_trainable_gradients_unchanged_by_the_image_gradient(pix, pattern):
    """bf16 rounding on: with some parameters training, pd, the loss and every trainable .grad are bit-identical to the same call with an
    img that does not require grad; frozen .grad are untouched."""
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(7)
    _, first, actions = batch(g, 2, 8)
    img = float_img(g, (2, 8, 32, 32, 3))
    res = []
    for want in (False, True):
        pol = copy.deepcopy(pol0).set_autograd(True)
        pre = freeze(pol, pattern) if pattern != "all" else {}
        x = img.clone().requires_grad_(want)
        (pd, _, _), st = pol({"img": x}, first, pol.initial_state(2))
        loss = bc_loss(pol, pd, actions)
        loss.backward()
        res.append((loss.detach(), pd, st, _grads(pol), pre, x.grad))
    (l0, pd0, s0, g0, _, x0), (l1, pd1, s1, g1, pre, x1) = res
    assert x0 is None and x1 is not None and x1.abs().sum() > 0
    assert torch.equal(l0, l1) and all(torch.equal(pd0[k], pd1[k]) for k in pd0)
    assert_same_state(s0, s1)
    for n in g0:
        if n in pre:
            assert (g1[n] is None and pre[n] is None) or torch.equal(g1[n], pre[n]), n
        else:
            assert (g0[n] is None) == (g1[n] is None) and (g0[n] is None or torch.equal(g0[n], g1[n])), n


def test_all_training_image_gradient_is_autograds(pix, exact):
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(8)
    _, first, actions = batch(g, 2, 4)
    img = float_img(g, (2, 4, 32, 32, 3)).requires_grad_(True)
    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(2))
    bc_loss(pol, pd, actions).backward()
    ref, leaf = oracle_img_grad(sd, cfg, img, first, lambda p: -O.logprob(p, actions).mean(), train=True)
    assert rel(img.grad, ref) < 5e-2
    for n, p in pol.named_parameters():
        if leaf[n].grad is not None and leaf[n].grad.any():
            assert rel(p.grad, leaf[n].grad) < 5e-2, n


def test_state_grad_window_gives_each_call_its_image_gradient(pix, exact):
    """A two-call window with the state attached and one backward: each call's frames are their own leaf and get autograd's gradient."""
    pol, sd, cfg = make_policy(small_kwargs())
    freeze_all(pol)
    pol.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(9)
    _, first, _ = batch(g, 2, 4)
    imgs = [float_img(g, (2, 4, 32, 32, 3)).requires_grad_(True) for _ in range(2)]
    leaf = {k: v.clone() for k, v in sd.items()}
    xs = [x.detach().clone().requires_grad_(True) for x in imgs]
    st, st_o, loss, loss_o = pol.initial_state(2), O.initial_state(cfg, 2), 0.0, 0.0
    for x, xo in zip(imgs, xs):
        (pd, _, _), st = pol({"img": x}, first, st)
        (pd_o, _, _), st_o = O.agent_policy_forward(leaf, cfg, xo, first, st_o)
    # the loss on the last call only: the first call's frames get their gradient through the KV memory
    camera_loss(pd).backward()
    camera_loss(pd_o).backward()
    for x, xo in zip(imgs, xs):
        assert rel(x.grad, xo.grad) < 5e-2


def test_backward_ops_with_and_without_the_image_gradient(pix, monkeypatch):
    """uint8 frames: the launch sequence of `loss.backward()` is unchanged (no image-gradient op).  All frozen with the image gradient:
    the backward runs firstconv_dimg and no weight-gradient op of the first conv."""
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(10)
    img, first, actions = batch(g, 2, 4)
    names = []
    for im, frozen in ((img, False), (img.float().requires_grad_(True), True)):
        pol = copy.deepcopy(pol0).set_autograd(True)
        if frozen:
            freeze_all(pol)
        with monkeypatch.context() as m:
            log = OpLog(m, _autograd_runner(pol))
            (pd, _, _), _ = pol({"img": im}, first, pol.initial_state(2))
            bc_loss(pol, pd, actions).backward()
        names.append(log.names())
    plain, pixel = names
    assert not any(n in IMG_OPS for n in plain)
    assert "firstconv_bwd" in plain
    assert pixel.count("firstconv_dimg") == 1 and "firstconv_bwd" not in pixel and "wgrad" not in pixel


def test_idm_backward_ops_with_the_image_gradient(pix, monkeypatch):
    idm, _, _ = make_idm()
    freeze_all(idm)
    idm.set_autograd(True)
    g = torch.Generator().manual_seed(11)
    _, first, actions = make_batch(g)
    img = float_img(g, (2, 8, 32, 32, 3)).requires_grad_(True)
    log = OpLog(monkeypatch, _autograd_runner(idm))
    (pd, _, _), _ = idm({"img": img}, first, idm.initial_state(2))
    (-O.logprob(pd, actions).mean()).backward()
    n = log.names()
    assert n.count("conv3d_t5_dimg") == 1 and "conv3d_t5_bwd" not in n and "wgrad" not in n


def test_pixel_emulation_mirrors_the_ops_api():
    """The image-gradient ops (ops_pixel.py, re-exported by ops) have an emulation with the same parameter names."""
    import inspect

    from video_pre_training_b200 import ops_pixel

    names = [n for n, fn in vars(ops_pixel).items() if not n.startswith("_") and inspect.isfunction(fn) and fn.__module__ == ops_pixel.__name__]
    assert sorted(names) == sorted(IMG_OPS)
    for name in names:
        assert getattr(ops, name) is getattr(ops_pixel, name)
        assert list(inspect.signature(getattr(ops_pixel, name)).parameters) == list(inspect.signature(getattr(emu_pixel_ops, name)).parameters)
