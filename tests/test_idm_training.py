"""IDM training step (IDMTrainer, video-pre-training_b200/training.py) on the CPU: the hand-written backward through the test-only torch
emulation of the ops (tests/emu_ops.py + tests/emu_idm_ops.py) against autograd through the oracle and through a forced replica of the
step's own tape.  tests/test_gpu_idm_training.py repeats it through the CUDA kernels."""
import inspect

import pytest
import torch

import emu_idm_ops
import emu_ops
import vpt_b200
import vpt_oracle as O
from common import perturb
from test_idm import SMALL_IDM
from video_pre_training_b200 import ops, ops_idm
from video_pre_training_b200.training import BCTrainer, IDMTrainer

# parameters whose gradient the reference's autograd sets to something other than a dense gradient (checked by pattern, not value)
NONE_PARAMS = ("net.lastlayer.",)          # computed, then discarded by the reference (lib/policy.py:390-391): None
ZERO_PARAMS = (".r_layer.weight", ".r_layer.bias")  # R meets the empty band of b_nd (10, 0): exact zeros
EMPTY_PARAMS = (".b_nd",)                  # the (10, 0) gradient


def kind(name):
    if name.startswith(NONE_PARAMS):
        return "none"
    if name.endswith(ZERO_PARAMS):
        return "zero"
    if name.endswith(EMPTY_PARAMS):
        return "empty"
    return "dense"


@pytest.fixture()
def emulated(monkeypatch):
    for mod in (emu_ops, emu_idm_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))
    yield


@pytest.fixture()
def exact(monkeypatch):
    """fp32 everywhere the kernels would store bf16: the emulated step is then the same function as the oracle."""
    from video_pre_training_b200 import policy, training

    for m in (emu_ops, policy, training):
        monkeypatch.setattr(m, "BF16", torch.float32)
    yield


def make_idm(seed=0, pert=True):
    torch.manual_seed(seed)
    kw = vpt_b200.idm_net_kwargs(**SMALL_IDM)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), kw)
    if pert:
        perturb(pol)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    cfg = O.Cfg(conv3d=True, **{k: v for k, v in kw.items() if k != "conv3d_params"})
    return pol, sd, cfg


def make_batch(g, B=2, T=8, hw=32):
    img = torch.randint(0, 256, (B, T, hw, hw, 3), dtype=torch.uint8, generator=g)
    actions = {"buttons": torch.randint(0, 2, (B, T, 20), generator=g), "camera": torch.randint(0, 11, (B, T, 2), generator=g)}
    return img, torch.zeros(B, T, dtype=torch.bool), actions


def oracle_grads(sd, cfg, img, first, actions):
    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    (pd, _, _), _ = O.idm_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, img.shape[0]))
    loss = -O.logprob(pd, actions).mean()
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaf.items()}


def run_case(calls=2, seed=0):
    pol, sd, cfg = make_idm()
    g = torch.Generator().manual_seed(seed)
    tr = IDMTrainer(pol)
    out = []
    for _ in range(calls):
        img, first, actions = make_batch(g)
        for p in pol.parameters():
            p.grad = None
        loss, st = tr.loss_and_grad(img, first, pol.initial_state(2), actions)
        assert st[0][0] is None and tuple(st[0][1][0].shape) == (2, 0, cfg.hidsize)
        loss_o, grads_o = oracle_grads(sd, cfg, img, first, actions)
        out.append((loss, loss_o, {n: p.grad for n, p in pol.named_parameters()}, grads_o))
    return out


def check_pattern(name, g):
    k = kind(name)
    if k == "none":
        assert g is None, name
    elif k == "zero":
        assert g is not None and g.dtype == torch.float32 and (g == 0).all(), name
    elif k == "empty":
        assert g is not None and tuple(g.shape) == (10, 0), name
    else:
        assert g is not None and g.dtype == torch.float32, f"no gradient for {name}"


def test_idm_backward_is_the_exact_gradient(emulated, exact):
    """bf16 rounding off: the hand-written backward must reproduce autograd through the oracle.  Outside the CNN to 1e-3 rel-L2; the
    CNN (and the conv3d) to the 5e-2 of the BC test, where an element that sits at a ReLU / max-pool boundary can flip its mask under the
    ~1e-6 difference between the folded forward and the oracle."""
    n_exact = 0
    for loss, loss_o, grads, grads_o in run_case():
        assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
        for n, g in grads.items():
            check_pattern(n, g)
            if kind(n) != "dense":
                continue
            g_o = grads_o[n]
            assert g_o is not None and g.shape == g_o.shape, n
            err = ((g - g_o).norm() / g_o.norm().clamp(min=1e-12)).item()
            cnn = n.startswith(("net.img_process.cnn.stacks", "net.conv3d_layer"))
            assert err < (5e-2 if cnn else 1e-3), (n, err)
            n_exact += not cnn
        # the oracle skips the empty relative term, so autograd through it leaves r_layer / b_nd without a gradient
        for n in grads_o:
            if kind(n) in ("zero", "empty"):
                assert grads_o[n] is None or not grads_o[n].any(), n
    assert n_exact > 30


def test_idm_step_with_bf16_rounding_points_emulated(emulated):
    """Every bf16 rounding point of the kernels emulated: mask flips against the fp32 oracle leave only the direction checkable
    (the BC test's criterion)."""
    for loss, loss_o, grads, grads_o in run_case(calls=1):
        assert abs(loss.item() - loss_o.item()) < 1e-2 * abs(loss_o.item())
        for n, g in grads.items():
            check_pattern(n, g)
            if kind(n) != "dense":
                continue
            g_o = grads_o[n]
            assert torch.isfinite(g).all()
            cos = (g * g_o).sum() / (g.norm() * g_o.norm()).clamp(min=1e-20)
            assert cos > 0.8, (n, cos.item())


def test_idm_backward_matches_autograd_at_the_taped_operating_point(emulated):
    """Autograd through the forced replica of the step's own tape (tests/forced_replica_idm.py) against the hand-written backward with
    every bf16 rounding point active: no mask can flip, so the bound is per parameter and as tight as the BC test's (2e-2).  A fixed
    CPU thread count makes the emulation's bf16 rounding independent of the host (see test_training.py)."""
    from forced_replica_idm import forced_loss_idm

    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    try:
        pol, sd, cfg = make_idm()
        img, first, actions = make_batch(torch.Generator().manual_seed(0))
        tr = IDMTrainer(pol)
        tr.keep_tape = True
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(2), actions)
        leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
        lf = forced_loss_idm(leaf, cfg, tr.last_tape, img, actions)
        lf.backward()
    finally:
        torch.set_num_threads(threads)
    assert abs(loss.item() - lf.item()) < 1e-4 * abs(lf.item())
    worst = {}
    for n, p in pol.named_parameters():
        check_pattern(n, p.grad)
        ref = leaf[n].grad
        if kind(n) == "none":
            assert ref is None, n  # the replica does not compute lastlayer either
            continue
        if kind(n) in ("zero", "empty"):
            assert ref is not None and ref.shape == p.grad.shape and not ref.any(), n  # the reference's autograd pattern
            continue
        worst[n] = ((p.grad - ref).norm() / ref.norm()).item()
    bad = {n: e for n, e in worst.items() if e > 2e-2}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


def test_idm_gradients_accumulate_over_calls(emulated):
    """Two calls without zeroing `.grad` give the sum of the two single-call gradients (accumulation over calls, like BCTrainer)."""
    pol, _, _ = make_idm()
    tr = IDMTrainer(pol)
    g = torch.Generator().manual_seed(5)
    batches = [make_batch(g, B=1) for _ in range(2)]
    single = []
    for img, first, actions in batches:
        for p in pol.parameters():
            p.grad = None
        tr.loss_and_grad(img, first, pol.initial_state(1), actions)
        single.append({n: None if p.grad is None else p.grad.clone() for n, p in pol.named_parameters()})
    for p in pol.parameters():
        p.grad = None
    for img, first, actions in batches:
        tr.loss_and_grad(img, first, pol.initial_state(1), actions)
    for n, p in pol.named_parameters():
        if single[0][n] is None:
            assert p.grad is None
            continue
        assert torch.allclose(p.grad, single[0][n] + single[1][n], rtol=1e-5, atol=1e-7), n


def test_idm_trainer_refuses_what_it_does_not_train():
    pol, _, _ = make_idm(pert=False)
    with pytest.raises(TypeError):
        IDMTrainer(pol.net)
    with pytest.raises(TypeError):
        BCTrainer(pol)  # unchanged: the policy trainer still refuses the IDM
    with pytest.raises(TypeError):
        IDMTrainer(vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(),
                                                 vpt_b200.policy_kwargs("1x", img_shape=[32, 32, 3], hidsize=256, attention_heads=2, timesteps=8,
                                                                        attention_memory_size=16, n_recurrence_layers=1),
                                                 vpt_b200.PI_HEAD_KWARGS))
    assert vpt_b200.IDMTrainer is IDMTrainer


def test_idm_frame_limit_is_enforced(emulated, monkeypatch):
    pol, _, _ = make_idm(pert=False)
    monkeypatch.setattr(pol.net, "idm_chunk_frames", 8)
    img, first, actions = make_batch(torch.Generator().manual_seed(0))
    with pytest.raises(NotImplementedError):
        IDMTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)


def test_idm_emulation_mirrors_the_ops_api():
    """The IDM backward ops (ops_idm.py, re-exported by ops) have an emulation with the same parameter names."""
    for name, fn in vars(ops_idm).items():
        if name.startswith("_") or not inspect.isfunction(fn) or fn.__module__ != ops_idm.__name__:
            continue
        assert getattr(ops, name) is fn, name
        emu = getattr(emu_idm_ops, name)
        assert list(inspect.signature(fn).parameters) == list(inspect.signature(emu).parameters), name


def test_conv3d_bwd_emulation_clips_time_per_sequence():
    """The emulated conv3d backward (the CPU reference of the GPU test) pads time per sequence: checked against a per-tap loop."""
    g = torch.Generator().manual_seed(1)
    B, T, H, W, C = 2, 3, 4, 4, 8
    img = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g)
    dy = emu_ops.to_zp(torch.randn(B * T, H, W, C, generator=g))
    dW, db = emu_idm_ops.conv3d_t5_bwd(img, dy, C)
    ref = torch.zeros(C, 5, 3, dtype=torch.float64)
    d = emu_ops.from_zp(dy).double().reshape(B, T, H * W, C)
    x = img.double().reshape(B, T, H * W, 3)
    for b in range(B):
        for t in range(T):
            for dt in range(5):
                tt = t + dt - 2
                if 0 <= tt < T:
                    ref[:, dt] += d[b, t].T @ x[b, tt]
    assert torch.allclose(dW.double(), ref.reshape(C, 15), rtol=1e-5, atol=1e-3)
    assert torch.allclose(db.double(), d.sum((0, 1, 2)), rtol=1e-5, atol=1e-4)
