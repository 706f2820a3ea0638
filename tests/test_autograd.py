"""The differentiable forward (`set_autograd`, training._AutogradRunner) on the CPU: `loss.backward()` through the test-only torch emulation
of the ops (tests/emu_ops.py, tests/emu_idm_ops.py, tests/emu_autograd_ops.py) against autograd through the oracle and against the
trainers.  tests/test_gpu_autograd.py repeats it through the CUDA kernels."""
import copy
import inspect

import pytest
import torch

import emu_autograd_ops
import emu_idm_ops
import emu_ops
import emu_rl_ops
import vpt_oracle as O
from common import make_policy, small_kwargs
from test_idm_training import check_pattern, kind, make_batch, make_idm
from video_pre_training_b200 import ops, ops_autograd
from video_pre_training_b200.policy import _autograd_runner
from video_pre_training_b200.training import BCTrainer, IDMTrainer, RLTrainer


def _with_grad(fn):
    """The emulation of some backward ops runs torch autograd itself; an autograd Function's backward runs with grad mode off."""
    def wrapped(*args, **kwargs):
        with torch.enable_grad():
            return fn(*args, **kwargs)
    return wrapped


@pytest.fixture()
def emulated(monkeypatch):
    for mod in (emu_ops, emu_idm_ops, emu_autograd_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                fn = getattr(mod, name)
                if name in ("maxpool3s2_bwd", "firstconv_bwd", "attention_bwd", "conv3d_t5_bwd"):
                    fn = _with_grad(fn)
                monkeypatch.setattr(ops, name, fn)
    yield


@pytest.fixture()
def exact(monkeypatch):
    """fp32 everywhere the kernels would store bf16: the emulated step is then the same function as the oracle."""
    from video_pre_training_b200 import policy, training

    for m in (emu_ops, policy, training):
        monkeypatch.setattr(m, "BF16", torch.float32)
    yield


def bc_loss(pol, pd, actions):
    return -pol.logprob(actions, pd).mean()


def custom_loss(pd, vpred, actions, pd_ref, denorm, target, kl_coef=0.3, ent_coef=0.05):
    """A loss on the camera head only: NLL - entropy bonus + kl_coef * KL(pd_ref || pd) + MSE on the denormalised value."""
    lp = pd["camera"]
    nll = -lp.gather(-1, actions["camera"].unsqueeze(-1)).squeeze(-1).sum(-1).mean()
    ent = -(torch.exp(lp) * lp).sum(-1).mean()
    kl = (torch.exp(pd_ref["camera"]) * (pd_ref["camera"] - lp)).sum(-1).mean()
    mse = ((denorm(vpred)[..., 0] - target) ** 2).mean()
    return nll - ent_coef * ent + kl_coef * kl + mse


def batch(g, B, T, reset=None):
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    if reset is not None:
        first[reset] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    return img, first, actions


def leaf_of(sd):
    return {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}


def compare(grads, grads_o, tol_cnn=5e-2, tol=1e-3):
    """Which parameters get None matches exactly; the rest to the BC test's rel-L2 bounds.  Returns the number of exact parameters."""
    n_exact = 0
    for n, g_o in grads_o.items():
        g = grads[n]
        assert (g is None) == (g_o is None), (n, g is None, g_o is None)
        if g_o is None:
            continue
        assert g.shape == g_o.shape and g.dtype == torch.float32, n
        if g_o.numel() == 0 or not g_o.any():
            assert not g.any(), n
            continue
        err = ((g - g_o).norm() / g_o.norm()).item()
        cnn = "img_process.cnn." in n or "conv3d_layer." in n
        assert err < (tol_cnn if cnn else tol), (n, err)
        n_exact += not cnn
    return n_exact


def test_bc_loss_backward_is_the_exact_gradient(emulated, exact):
    """bf16 rounding off: the BC loss through the differentiable forward, two chunks with carried state and an episode start mid-batch,
    equals autograd through the oracle; value_head.* gets None (the loss never touches vpred)."""
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(0)
    B, T = 2, 8
    st, st_o = pol.initial_state(B), O.initial_state(cfg, B)
    n_exact = 0
    for c in range(2):
        img, first, actions = batch(g, B, T, reset=(1, 3) if c == 1 else None)
        for p in pol.parameters():
            p.grad = None
        (pd, vpred, _), st = pol({"img": img}, first, st)
        assert vpred.requires_grad and all(not k.requires_grad for _, (k, v) in st)
        loss = bc_loss(pol, pd, actions)
        loss.backward()
        leaf = leaf_of(sd)
        (pd_o, _, _), st_o = O.agent_policy_forward(leaf, cfg, img, first, st_o)
        st_o = [(m, (k.detach(), v.detach())) for (m, (k, v)) in st_o]
        loss_o = -O.logprob(pd_o, actions).mean()
        loss_o.backward()
        assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
        grads = {n: p.grad for n, p in pol.named_parameters()}
        assert grads["value_head.linear.weight"] is None
        n_exact += compare(grads, {k: v.grad for k, v in leaf.items()})
    assert n_exact > 80


def test_custom_camera_loss_is_the_exact_gradient(emulated, exact):
    """An entropy bonus, the NLL and a KL on the camera head only, plus an MSE on denormalize(vpred): the buttons head gets None, the
    value head a dense gradient, everything else the oracle's."""
    pol, sd, cfg = make_policy(small_kwargs())
    ref, _, _ = make_policy(small_kwargs(), seed=3)
    sd_ref = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(1)
    B, T = 2, 8
    img, first, actions = batch(g, B, T, reset=(0, 2))
    target = 2.0 * torch.randn(B, T, generator=g)
    with torch.no_grad():
        (pd_ref, _, _), _ = O.agent_policy_forward(sd_ref, cfg, img, first, O.initial_state(cfg, B))
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    loss = custom_loss(pd, vpred, actions, pd_ref, pol.denormalize, target)
    loss.backward()
    leaf = leaf_of(sd)
    (pd_o, vpred_o, _), _ = O.agent_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, B))
    loss_o = custom_loss(pd_o, vpred_o, actions, pd_ref, pol.denormalize, target)
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    grads = {n: p.grad for n, p in pol.named_parameters()}
    assert grads["pi_head.buttons.linear_layer.weight"] is None and grads["value_head.linear.weight"].abs().sum() > 0
    assert compare(grads, {k: v.grad for k, v in leaf.items()}) > 40


def test_idm_loss_backward_is_the_exact_gradient(emulated, exact):
    """The IDM loss: lastlayer.* None, r_layer.* zeros, b_nd an empty (10, 0) gradient, the rest the oracle's (conv3d included)."""
    pol, sd, cfg = make_idm()
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(0)
    img, first, actions = make_batch(g)
    (pd, vpred, _), st = pol({"img": img}, first, pol.initial_state(2))
    assert vpred is None
    loss = -pol.logprob(actions, pd).mean()
    loss.backward()
    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    (pd_o, _, _), _ = O.idm_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    loss_o = -O.logprob(pd_o, actions).mean()
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    grads = {n: p.grad for n, p in pol.named_parameters()}
    special = {n for n in grads if kind(n) != "dense"}
    for n in special:  # the IDMTrainer's pattern (tests/test_idm_training.py)
        check_pattern(n, grads[n])
    assert compare({n: g for n, g in grads.items() if n not in special}, {k: v.grad for k, v in leaf.items() if k not in special}) > 20


def _grads(pol):
    return {n: None if p.grad is None else p.grad.clone() for n, p in pol.named_parameters()}


def _worst(a, b):
    worst = 0.0
    for n in a:
        assert (a[n] is None) == (b[n] is None), n
        if a[n] is not None and b[n].any():
            worst = max(worst, ((a[n] - b[n]).norm() / b[n].norm()).item())
    return worst


def test_bc_and_idm_losses_match_the_trainers(emulated):
    """Every bf16 rounding point active: the BC and IDM losses through `loss.backward()` against BCTrainer / IDMTrainer on the same batch
    (the same forward; the logits gradient differs by bf16 rounding of the upstream gradient only)."""
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(2)
    img, first, actions = batch(g, 2, 8, reset=(1, 4))
    loss_t, _ = BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
    ref = _grads(pol)
    pol.zero_grad(set_to_none=True)
    (pd, _, _), _ = pol.set_autograd(True)({"img": img}, first, pol.initial_state(2))
    loss = bc_loss(pol, pd, actions)
    loss.backward()
    assert abs(loss.item() - loss_t.item()) < 1e-6 * abs(loss_t.item())
    assert _worst(_grads(pol), ref) < 1e-2

    idm, _, _ = make_idm()
    img, first, actions = make_batch(g)
    IDMTrainer(idm).loss_and_grad(img, first, idm.initial_state(2), actions)
    ref = _grads(idm)
    idm.zero_grad(set_to_none=True)
    (pd, _, _), _ = idm.set_autograd(True)({"img": img}, first, idm.initial_state(2))
    (-idm.logprob(actions, pd).mean()).backward()
    assert _worst(_grads(idm), ref) < 1e-2


def test_trainers_and_differentiable_forward_share_the_layouts(emulated, monkeypatch):
    """BCTrainer, RLTrainer and `loss.backward()` on one policy read the policy's one forward fold and net backward copy, rebuilt once for
    all three after an in-place parameter update, and get the same gradients as each of them on a copy of the policy of its own."""
    for name in dir(emu_rl_ops):
        if not name.startswith("_") and callable(getattr(emu_rl_ops, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(emu_rl_ops, name))
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(9)
    B, T = 2, 8
    img, first, actions = batch(g, B, T)
    rl_args = (0.1 * torch.randn(B, T, generator=g) - 14.0, torch.randn(B, T, generator=g), 3.0 + torch.randn(B, T, generator=g))
    runs = []
    for pols in ([pol0] * 3, [copy.deepcopy(pol0) for _ in range(3)]):
        bc, rl, ag = BCTrainer(pols[0]), RLTrainer(pols[1]), _autograd_runner(pols[2].set_autograd(True))
        for tr in (bc, rl, ag):
            tr.keep_tape = True
        rounds = []
        for _ in range(2):
            grads = []
            for i, pol in enumerate(pols):
                pol.zero_grad(set_to_none=True)
                if i == 0:
                    bc.loss_and_grad(img, first, pol.initial_state(B), actions)
                elif i == 1:
                    rl.loss_and_grad(img, first, pol.initial_state(B), actions, *rl_args, vf_coef=0.5, kl_coef=0.0)
                else:
                    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
                    bc_loss(pol, pd, actions).backward()
                grads.append(_grads(pol))
            rounds.append((grads, [(tr.last_tape["prep"], tr.last_tape["wts"]) for tr in (bc, rl, ag)]))
            with torch.no_grad():
                for pol in {id(p): p for p in pols}.values():
                    for p in pol.parameters():
                        if p.requires_grad:
                            p.mul_(0.99)
        runs.append(rounds)
    for (grads, layouts), (grads_apart, _) in zip(*runs):
        assert all(a is b for lay in layouts[1:] for a, b in zip(lay, layouts[0]))
        for gs, ga in zip(grads, grads_apart):
            assert gs.keys() == ga.keys()
            for n in gs:
                assert (gs[n] is None and ga[n] is None) or torch.equal(gs[n], ga[n]), n
    (_, first_layouts), (_, second_layouts) = runs[0]
    assert all(a is not b for a, b in zip(first_layouts[0], second_layouts[0]))


def test_bare_network_latent_is_differentiable(emulated, exact):
    """MinecraftPolicy on its own: the latent is attached to the graph and its gradient matches the oracle's through the agent policy's
    latent (the heads' parameters are not the network's)."""
    pol, sd, cfg = make_policy(small_kwargs())
    net = pol.net.set_autograd(True)
    g = torch.Generator().manual_seed(5)
    img, first, _ = batch(g, 1, 8)
    w = torch.randn(1, 8, cfg.hidsize, generator=g)
    (lat, lat2), _ = net({"img": img}, net.initial_state(1), {"first": first})
    assert lat is lat2 and lat.requires_grad
    (lat * w).sum().backward()
    leaf = leaf_of(sd)
    lat_o, _ = O.minecraft_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 1))
    (lat_o * w).sum().backward()
    grads_o = {k[4:]: v.grad for k, v in leaf.items() if k.startswith("net.")}
    assert compare({n: p.grad for n, p in net.named_parameters()}, grads_o) > 30


def test_inference_path_is_untouched(emulated):
    """Flag off, no_grad, or every parameter frozen: bit-identical outputs, no grad_fn, no tape."""
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(6)
    img, first, _ = batch(g, 1, 8)
    (pd0, v0, _), st0 = pol({"img": img}, first, pol.initial_state(1))
    assert v0.grad_fn is None and pol._ag_runner is None
    pol.set_autograd(True)
    with torch.no_grad():
        (pd1, v1, _), _ = pol({"img": img}, first, pol.initial_state(1))
    with torch.inference_mode():
        (pd3, v3, _), _ = pol({"img": img}, first, pol.initial_state(1))
    for p in pol.parameters():
        p.requires_grad_(False)
    (pd2, v2, _), st2 = pol({"img": img}, first, pol.initial_state(1))
    assert pol._ag_runner is None
    for pd, v in ((pd1, v1), (pd2, v2), (pd3, v3)):
        assert v.grad_fn is None and torch.equal(v, v0)
        for k in pd0:
            assert pd[k].grad_fn is None and torch.equal(pd[k], pd0[k])
    assert pol.act({"img": img[:, 0]}, first[:, 0], pol.initial_state(1))[2]["vpred"].grad_fn is None


def test_logprob_values_do_not_change(emulated):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(7)
    img, first, actions = batch(g, 1, 8)
    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(1))
    lp0 = pol.logprob(actions, pd)
    (pd, _, _), _ = pol.set_autograd(True)({"img": img}, first, pol.initial_state(1))
    lp1 = pol.logprob(actions, pd)
    assert not lp0.requires_grad and lp1.requires_grad
    assert torch.equal(lp1.detach(), pol.logprob(actions, {k: v.detach() for k, v in pd.items()}))


def test_refusals(emulated):
    pol, _, _ = make_policy(small_kwargs())
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(8)
    img, first, actions = batch(g, 1, 8)
    st = pol.initial_state(1)
    with pytest.raises(NotImplementedError):  # the fp32-parity mode does not train
        pol.set_precision("fp32")({"img": img}, first, st)
    pol.set_precision("bf16")
    big = torch.zeros(1, pol.net.cnn_chunk_frames + 1, 32, 32, 3, dtype=torch.uint8)
    with pytest.raises(NotImplementedError):
        pol({"img": big}, torch.zeros(1, big.shape[1], dtype=torch.bool), st)
    bad = [(m, (k.clone().requires_grad_(True), v)) for m, (k, v) in st]
    with pytest.raises(ValueError):  # no gradient through the KV memory
        pol({"img": img}, first, bad)
    assert pol._ag_runner is None or pol._ag_runner.last_tape is None

    (pd, _, _), _ = pol({"img": img}, first, st)
    loss = bc_loss(pol, pd, actions)
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="once"):
        loss.backward()

    (pd, _, _), _ = pol({"img": img}, first, st)
    with torch.no_grad():
        pol.net.final_ln.weight.add_(0.01)
    with pytest.raises(RuntimeError):  # torch's version check: a parameter changed between forward and backward
        bc_loss(pol, pd, actions).backward()

    for p in pol.parameters():
        p.grad = None
    (pd, _, _), _ = pol({"img": img}, first, st)
    with pytest.raises(NotImplementedError):
        torch.autograd.grad(bc_loss(pol, pd, actions), [pol.net.final_ln.weight], create_graph=True)

    idm, _, _ = make_idm()
    idm.set_autograd(True)
    big = torch.zeros(5, 128, 32, 32, 3, dtype=torch.uint8)
    with pytest.raises(NotImplementedError):
        idm({"img": big}, torch.zeros(5, 128, dtype=torch.bool), idm.initial_state(5))


def test_emulation_mirrors_the_ops_api():
    for name, fn in vars(ops_autograd).items():
        if name.startswith("_") or not inspect.isfunction(fn) or fn.__module__ != ops_autograd.__name__:
            continue
        assert getattr(ops, name) is fn, name
        assert list(inspect.signature(fn).parameters) == list(inspect.signature(getattr(emu_autograd_ops, name)).parameters), name
