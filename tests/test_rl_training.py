"""RL fine-tuning step (RLTrainer, video-pre-training_b200/training.py) on the CPU: the hand-written backward through the test-only torch
emulation of the ops (tests/emu_ops.py + tests/emu_rl_ops.py) against autograd of the loss through the oracle.
tests/test_gpu_rl_training.py repeats it through the CUDA kernels."""
import inspect

import pytest
import torch

import emu_ops
import emu_rl_ops
import vpt_b200
import vpt_oracle as O
from common import make_policy, perturb, small_kwargs
from video_pre_training_b200 import ops, ops_rl
from video_pre_training_b200.training import BCTrainer, RLTrainer

NORM = ("running_mean", "running_mean_sq", "debiasing_term")
# ratio targets of the batch rows: clipped on both sides, unclipped inside and outside the band, none on a boundary of clip = 0.2
RATIOS = (0.5, 0.7, 0.9, 1.0, 1.1, 1.35, 1.6, 0.75)
ADV_SIGNS = (1.0, -1.0, 1.0, -1.0, -1.0, 1.0, -1.0, -1.0)


@pytest.fixture()
def emulated(monkeypatch):
    for mod in (emu_ops, emu_rl_ops):
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


def ewma_normalize(norm, x, beta=0.99999):
    """NormalizeEwma.forward in training mode (lib/normalize_ewma.py:36-55, norm_axes=2): updates `norm` in place, returns the
    normalised x."""
    with torch.no_grad():
        d = x.detach().float()
        bm, bsq = d.mean(dim=(0, 1)), (d ** 2).mean(dim=(0, 1))
        norm["running_mean"].mul_(beta).add_(bm * (1.0 - beta))
        norm["running_mean_sq"].mul_(beta).add_(bsq * (1.0 - beta))
        norm["debiasing_term"].mul_(beta).add_(1.0 * (1.0 - beta))
    deb = norm["debiasing_term"].clamp(min=1e-5)
    mean = norm["running_mean"] / deb
    var = (norm["running_mean_sq"] / deb - mean ** 2).clamp(min=1e-2)
    return (x - mean[None, None]) / torch.sqrt(var)[None, None]


def rl_loss(pd, vpred, actions, old_lp, adv, returns, pd_ref, norm, vf_coef, kl_coef, clip):
    """The issue's loss from the reference's pieces: get_logprob_of_action, ScaledMSEHead.loss (training mode), get_kl_of_action_dists."""
    lp = O.logprob(pd, actions)
    ratio = torch.exp(lp - old_lp)
    l_pi = -torch.min(ratio * adv, ratio.clamp(1 - clip, 1 + clip) * adv).mean()
    l_v = ((vpred - ewma_normalize(norm, returns[..., None])) ** 2).mean()
    loss = l_pi + vf_coef * l_v
    if pd_ref is not None:
        kl = sum((torch.exp(pd_ref[k]) * (pd_ref[k] - pd[k])).sum(-1).sum(-1) for k in pd)
        loss = loss + kl_coef * kl.mean()
    return loss


def ref_pd(cfg, sd_ref, img, first, state):
    with torch.no_grad():
        (pd, _, _), st = O.agent_policy_forward(sd_ref, cfg, img, first, state)
    return pd, [(m, (k.detach(), v.detach())) for (m, (k, v)) in st]


def make_rl_batch(g, lp, B, T):
    """old_logprob placing each row's ratio at RATIOS (given the current log-probs lp), advantages with the signs ADV_SIGNS, returns."""
    r = torch.tensor(RATIOS).repeat(B * T // len(RATIOS) + 1)[: B * T].reshape(B, T)
    s = torch.tensor(ADV_SIGNS).repeat(B * T // len(ADV_SIGNS) + 1)[: B * T].reshape(B, T)
    old = (lp - torch.log(r)).float()
    adv = (s * (0.5 + torch.rand(B, T, generator=g))).float()
    returns = (3.0 + 2.0 * torch.randn(B, T, generator=g)).float()
    return old, adv, returns


def make_pair(seed=0):
    pol, sd, cfg = make_policy(small_kwargs(), seed=seed)
    ref, sd_ref, _ = make_policy(small_kwargs(), seed=seed)
    perturb(ref, seed=7)  # the frozen reference policy: the same initial weights, perturbed differently
    sd_ref = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    return pol, sd, sd_ref, cfg


def run_rl_case(B=2, T=8, chunks=2, vf_coef=0.5, kl_coef=0.1, clip=0.2, with_ref=True, seed=0):
    """Two chunks with carried state; chunk 1 has an episode start in row 1 mid-batch (at t = 3)."""
    pol, sd, sd_ref, cfg = make_pair()
    g = torch.Generator().manual_seed(seed)
    tr = RLTrainer(pol)
    st, st_o, st_r = pol.initial_state(B), O.initial_state(cfg, B), O.initial_state(cfg, B)
    norm = {k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM}
    out = []
    for c in range(chunks):
        img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
        first = torch.zeros(B, T, dtype=torch.bool)
        if c == 1:
            first[1, 3] = True
        actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
        pd_ref, st_r = ref_pd(cfg, sd_ref, img, first, st_r) if with_ref else (None, None)
        with torch.no_grad():
            (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, st_o)
        old, adv, returns = make_rl_batch(g, O.logprob(pd0, actions), B, T)
        for p in pol.parameters():
            p.grad = None
        loss, st = tr.loss_and_grad(img, first, st, actions, old, adv, returns, pd_ref, vf_coef=vf_coef, kl_coef=kl_coef, clip=clip)
        leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}
        (pd, vpred, _), st_o = O.agent_policy_forward(leaf, cfg, img, first, st_o)
        st_o = [(m, (k.detach(), v.detach())) for (m, (k, v)) in st_o]
        loss_o = rl_loss(pd, vpred, actions, old, adv, returns, pd_ref, norm, vf_coef, kl_coef, clip)
        loss_o.backward()
        ratio = torch.exp(O.logprob(pd0, actions) - old)
        out.append(dict(loss=loss, loss_o=loss_o.detach(), grads={n: p.grad for n, p in pol.named_parameters()},
                        grads_o={k: v.grad for k, v in leaf.items()}, norm={k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM},
                        norm_o={k: v.clone() for k, v in norm.items()}, stats={k: v.item() for k, v in tr.stats.items()}, ratio=ratio, adv=adv))
    return out


def test_rl_backward_is_the_exact_gradient(emulated, exact):
    """bf16 rounding off: the hand-written RL backward equals autograd of the loss through the oracle, the value head included, and the
    normaliser holds the reference's values after every call.  Outside the CNN to 1e-3 rel-L2, inside it to 5e-2 (mask flips, see
    test_training.py)."""
    n_exact = 0
    for o in run_rl_case():
        lo, hi = 1 - 0.2, 1 + 0.2
        r, a = o["ratio"], o["adv"]
        clipped = ((a > 0) & (r > hi)) | ((a < 0) & (r < lo))
        assert 0 < clipped.sum() < clipped.numel() and ((a > 0) & (r > hi)).any() and ((a < 0) & (r < lo)).any()
        assert ((r - hi).abs() > 1e-3).all() and ((r - lo).abs() > 1e-3).all()
        assert abs(o["stats"]["clipfrac"] - clipped.float().mean().item()) < 1e-6
        assert abs(o["loss"].item() - o["loss_o"].item()) < 1e-4 * abs(o["loss_o"].item())
        for k in NORM:
            assert torch.allclose(o["norm"][k], o["norm_o"][k], rtol=1e-6, atol=0), k
        for n, g in o["grads"].items():
            g_o = o["grads_o"][n]
            if n.startswith("value_head.normalizer."):
                assert g is None and g_o is None
                continue
            assert g is not None and g_o is not None and g.shape == g_o.shape and g.dtype == torch.float32, n
            err = ((g - g_o).norm() / g_o.norm().clamp(min=1e-12)).item()
            cnn = n.startswith("net.img_process.cnn")  # (the ImpalaCNN includes its dense layer, as in test_training.py)
            assert err < (5e-2 if cnn else 1e-3), (n, err)
            n_exact += not cnn
        assert o["grads"]["value_head.linear.weight"].abs().sum() > 0
    assert n_exact > 80


def test_rl_without_reference_policy(emulated, exact):
    """pd_ref = None (kl_coef = 0): the KL term and its statistic vanish, the rest is still the exact gradient."""
    for o in run_rl_case(chunks=1, kl_coef=0.0, with_ref=False):
        assert o["stats"]["kl_ref"] == 0.0
        assert abs(o["loss"].item() - o["loss_o"].item()) < 1e-4 * abs(o["loss_o"].item())
        for n in ("value_head.linear.weight", "pi_head.buttons.linear_layer.weight", "net.final_ln.weight"):
            g, g_o = o["grads"][n], o["grads_o"][n]
            assert ((g - g_o).norm() / g_o.norm()).item() < 1e-3, n


def test_rl_with_unit_ratio_and_advantage_is_the_bc_step(emulated, exact):
    """A = 1, old_logprob = the step's own log-probs, vf_coef = kl_coef = 0: c[r] = 1/N, i.e. the BC gradient; the value head's is 0."""
    pol, sd, _, cfg = make_pair()
    g = torch.Generator().manual_seed(3)
    B, T = 2, 8
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
    lp = pol.logprob(actions, pd).reshape(B, T).float()
    BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(B), actions)
    bc = {n: None if p.grad is None else p.grad.clone() for n, p in pol.named_parameters()}
    for p in pol.parameters():
        p.grad = None
    ones = torch.ones(B, T)
    RLTrainer(pol).loss_and_grad(img, first, pol.initial_state(B), actions, lp, ones, torch.zeros(B, T), None, vf_coef=0.0, kl_coef=0.0)
    for n, p in pol.named_parameters():
        if n.startswith("value_head.linear."):
            assert bc[n] is None and p.grad is not None and not p.grad.any(), n
        elif bc[n] is None:
            assert p.grad is None, n
        else:
            assert ((p.grad - bc[n]).norm() / bc[n].norm()).item() < 1e-5, n


def test_rl_second_call_keeps_the_policy_weight_layouts(emulated):
    """The normaliser update of a call does not invalidate the kernel-layout weight caches, but `denormalize` sees it."""
    pol, _, _, _ = make_pair()
    tr = RLTrainer(pol)
    g = torch.Generator().manual_seed(4)
    B, T = 1, 8
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    args = (torch.zeros(B, T), torch.ones(B, T), 5.0 + torch.randn(B, T, generator=g))
    tr.loss_and_grad(img, first, pol.initial_state(B), actions, *args, vf_coef=1.0, kl_coef=0.0)
    layouts = lambda: (pol.net.prepared(), pol._heads_prepared(), pol.net.prepared_backward(), pol._heads_prepared_backward(tr._head_layers()))
    held = layouts()
    v0 = pol.denormalize(torch.zeros(1, 1, 1)).clone()
    tr.loss_and_grad(img, first, pol.initial_state(B), actions, *args[:2], args[2] + 3.0, vf_coef=1.0, kl_coef=0.0)
    assert all(a is b for a, b in zip(layouts(), held))
    assert not torch.equal(pol.denormalize(torch.zeros(1, 1, 1)), v0)


def test_rl_trainer_refuses_bad_input():
    pol, _, _ = make_policy(small_kwargs(), pert=False)
    with pytest.raises(TypeError):
        RLTrainer(pol.net)
    idm = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0),
                                       vpt_b200.idm_net_kwargs(img_shape=[32, 32, 128], hidsize=256, attention_heads=2, timesteps=8,
                                                               attention_memory_size=8, n_recurrence_layers=1, impala_width=4))
    with pytest.raises(TypeError):
        RLTrainer(idm)
    tr = RLTrainer(pol)
    B, T = 1, 8
    img = torch.zeros(B, T, 32, 32, 3, dtype=torch.uint8)
    first = torch.zeros(B, T, dtype=torch.bool)
    actions = {"camera": torch.zeros(B, T, 1, dtype=torch.long), "buttons": torch.zeros(B, T, 1, dtype=torch.long)}
    z = torch.zeros(B, T)
    with pytest.raises(ValueError):  # a KL penalty needs the reference policy's distributions
        tr.loss_and_grad(img, first, pol.initial_state(B), actions, z, z, z, None, vf_coef=0.5, kl_coef=0.1)
    with pytest.raises(ValueError):
        tr.loss_and_grad(img, first, pol.initial_state(B), actions, z.double(), z, z, vf_coef=0.5, kl_coef=0.0)
    with pytest.raises(ValueError):
        tr.loss_and_grad(img, first, pol.initial_state(B), actions, z, z[:, :4], z, vf_coef=0.5, kl_coef=0.0)
    with pytest.raises(TypeError):  # the coefficients have no default
        tr.loss_and_grad(img, first, pol.initial_state(B), actions, z, z, z)
    assert all(p.grad is None for p in pol.parameters())
    assert vpt_b200.RLTrainer is RLTrainer


def test_rl_emulation_mirrors_the_ops_api():
    for name, fn in vars(ops_rl).items():
        if name.startswith("_") or not inspect.isfunction(fn) or fn.__module__ != ops_rl.__name__:
            continue
        assert getattr(ops, name) is fn, name
        assert list(inspect.signature(fn).parameters) == list(inspect.signature(getattr(emu_rl_ops, name)).parameters), name


def rl_vs_forced(pol, sd, cfg, tr, img, first, actions, old, adv, returns, pd_ref, norm0, vf_coef, kl_coef, clip=0.2):
    """Per-parameter rel-L2 of the step's gradients against autograd through the forced replica of its own tape (tests/forced_replica_rl.py)."""
    from forced_replica_rl import forced_rl_loss

    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}
    lf = forced_rl_loss(leaf, cfg, tr.last_tape, img, first, actions, old, adv, returns, pd_ref, norm0, vf_coef, kl_coef, clip)
    lf.backward()
    worst = {}
    for n, p in pol.named_parameters():
        if n.startswith("value_head.normalizer."):
            continue
        worst[n] = ((p.grad - leaf[n].grad).norm() / leaf[n].grad.norm()).item()
    return lf.item(), worst


def test_rl_backward_matches_autograd_at_the_taped_operating_point(emulated):
    """Every bf16 rounding point active, against the forced replica: no mask can flip, so the bound is per parameter (BC's 2e-2)."""
    threads = torch.get_num_threads()
    torch.set_num_threads(8)  # (the CPU convolutions' summation order, see test_training.py)
    try:
        pol, sd, sd_ref, cfg = make_pair()
        g = torch.Generator().manual_seed(0)
        B, T = 2, 8
        img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
        first = torch.zeros(B, T, dtype=torch.bool)
        first[1, 3] = True
        actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
        pd_ref, _ = ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, B))
        with torch.no_grad():
            (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, B))
        old, adv, returns = make_rl_batch(g, O.logprob(pd0, actions), B, T)
        norm0 = {k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM}
        tr = RLTrainer(pol)
        tr.keep_tape = True
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)
        lf, worst = rl_vs_forced(pol, sd, cfg, tr, img, first, actions, old, adv, returns, pd_ref, norm0, 0.5, 0.1)
    finally:
        torch.set_num_threads(threads)
    # (the step's vpred comes from the bf16 value-head weights of the inference kernels, the replica's from the fp32 ones)
    assert abs(loss.item() - lf) < 1e-3 * abs(lf)
    bad = {n: e for n, e in worst.items() if e > 2e-2}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]
