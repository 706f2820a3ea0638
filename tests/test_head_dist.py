"""`pi_head` (policy.py `_DictActionHead` / `_CategoricalActionHead`) on the CPU through the test-only emulation of the ops
(tests/emu_ops.py, emu_rl_ops.py, emu_dist_ops.py): the reference's distribution methods (lib/action_head.py:136-260) with their shapes,
dtypes and values, the autograd wiring against float64 autograd of the reference formulas, the entropy bonus of `RLTrainer`, and the
unchanged `state_dict` keys.  tests/test_gpu_head_dist.py runs the kernels."""
import copy
import os

import pytest
import torch

import emu_dist_ops
import emu_ops
import emu_rl_ops
import refshim
import vpt_b200
import vpt_oracle as O
from common import small_kwargs
from test_rl_training import NORM, make_pair, make_rl_batch, ref_pd, rl_loss
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import _CategoricalActionHead, _DictActionHead
from video_pre_training_b200.training import RLTrainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPACES = {  # name -> [(head, shape, n)] in the action space's order (types.py)
    "agent": [("camera", (1,), 121), ("buttons", (1,), 8641)],
    "idm": [("buttons", (20,), 2), ("camera", (2,), 11)],
}


@pytest.fixture()
def emulated(monkeypatch):
    for mod in (emu_ops, emu_rl_ops, emu_dist_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))
    yield


@pytest.fixture()
def exact(monkeypatch):
    from video_pre_training_b200 import policy, training

    for m in (emu_ops, policy, training):
        monkeypatch.setattr(m, "BF16", torch.float32)
    yield


def our_head(space):
    head = _DictActionHead()
    for name, shape, n in SPACES[space]:
        head.add_module(name, _CategoricalActionHead(shape, n))
    return head


def ref_head(space):
    if not refshim.available():
        pytest.skip("the reference checkout is not present")
    refshim.load()
    import lib.action_head as AH
    from gym3.types import DictType, Discrete, TensorType

    ac = DictType(**{name: TensorType(Discrete(n), shape) for name, shape, n in SPACES[space]})
    return AH.make_action_head(ac, 8, temperature=2.0)


def make_pd(space, B=3, T=5, seed=0, masked=True, dtype=torch.float32):
    """Log-probs as the policy's forward makes them: log_softmax of logits, masked entries -100 before it (lib/action_head.py:170-171)."""
    g = torch.Generator().manual_seed(seed)
    pd = {}
    for name, shape, n in SPACES[space]:
        x = 3.0 * torch.randn(B, T, *shape, n, generator=g)
        if masked:
            x[torch.rand(x.shape, generator=g) < 0.3] = -100.0
        pd[name] = torch.log_softmax(x, -1).to(dtype)
    return pd


def actions_for(space, B=3, T=5, seed=1):
    g = torch.Generator().manual_seed(seed)
    return {name: torch.randint(0, n, (B, T, *shape), generator=g) for name, shape, n in SPACES[space]}


def ref_entropy(pd):
    return sum(-(torch.exp(v) * v).sum(-1).flatten(2).sum(-1) for v in pd.values())


def ref_kl(pq, pp):
    return sum((torch.exp(pq[k]) * (pq[k] - pp[k])).sum(-1).flatten(2).sum(-1, keepdim=True) for k in pq)


@pytest.mark.parametrize("space", list(SPACES))
@pytest.mark.parametrize("masked", [False, True])
def test_distribution_methods_match_the_reference(emulated, space, masked):
    ours, ref = our_head(space), ref_head(space)
    pq, pp = make_pd(space, seed=0, masked=masked), make_pd(space, seed=1, masked=masked)
    ac = actions_for(space)
    for name, got, want in (("entropy", ours.entropy(pq), ref.entropy(pq)), ("kl", ours.kl_divergence(pq, pp), ref.kl_divergence(pq, pp)),
                            ("logprob", ours.logprob(ac, pq), ref.logprob(ac, pq))):
        assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape)
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), (name, (got - want).abs().max().item())
    for k, sub in ours.items():  # the sub-heads on their own
        assert sub.entropy(pq[k]).shape == ref[k].entropy(pq[k]).shape
        assert torch.allclose(sub.entropy(pq[k]), ref[k].entropy(pq[k]), rtol=1e-5, atol=1e-5), k
        assert torch.allclose(sub.kl_divergence(pq[k], pp[k]), ref[k].kl_divergence(pq[k], pp[k]), rtol=1e-5, atol=1e-5), k
        assert torch.equal(sub.logprob(ac[k], pq[k]), ref[k].logprob(ac[k], pq[k])), k
    for det in (False, True):
        torch.manual_seed(11)
        a = ours.sample(pq, det)
        torch.manual_seed(11)
        b = ref.sample(pq, det)
        assert list(a) == list(b)
        for k in a:
            assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), (k, det)


@pytest.mark.parametrize("space", list(SPACES))
def test_values_and_shapes_without_the_reference(emulated, space):
    """The reference's formulas restated in float64 (this runs where the reference checkout is absent too)."""
    head = our_head(space)
    pq, pp = make_pd(space, seed=2), make_pd(space, seed=3)
    d = lambda pd: {k: v.double() for k, v in pd.items()}
    ent, kl = head.entropy(pq), head.kl_divergence(pq, pp)
    assert ent.shape == (3, 5) and kl.shape == (3, 5, 1) and ent.dtype == kl.dtype == torch.float32
    assert torch.allclose(ent.double(), ref_entropy(d(pq)), rtol=1e-5, atol=1e-5)
    assert torch.allclose(kl.double(), ref_kl(d(pq), d(pp)), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("space", list(SPACES))
def test_autograd_matches_float64_autograd_of_the_reference_formulas(emulated, monkeypatch, space):
    head = our_head(space)
    g = torch.Generator().manual_seed(5)
    wq, wp = make_pd(space, seed=6), make_pd(space, seed=7)
    leaf = lambda pd, dt: {k: v.detach().to(dt).requires_grad_(True) for k, v in pd.items()}
    q32, p32, q64, p64 = leaf(wq, torch.float32), leaf(wp, torch.float32), leaf(wq, torch.float64), leaf(wp, torch.float64)
    we, wk = torch.randn(3, 5, generator=g), torch.randn(3, 5, 1, generator=g)
    ((head.entropy(p32) * we).sum() + (head.kl_divergence(q32, p32) * wk).sum()).backward()
    ((ref_entropy(p64) * we.double()).sum() + (ref_kl(q64, p64) * wk.double()).sum()).backward()
    for k in wq:
        for a, b in ((q32[k], q64[k]), (p32[k], p64[k])):
            assert a.grad.dtype == torch.float32
            err = ((a.grad.double() - b.grad).norm() / b.grad.norm()).item()
            assert err < 1e-5, (k, err)
    # one side only: the backward kernel is asked for that side alone, and the other input gets no gradient
    wants = []
    monkeypatch.setattr(ops, "head_kl_bwd", lambda lq, lp, g, groups=1, want_q=True, want_p=True: wants.append((want_q, want_p))
                        or emu_dist_ops.head_kl_bwd(lq, lp, g, groups, want_q, want_p))
    for side in ("q", "p"):
        wants.clear()
        q = leaf(wq, torch.float32) if side == "q" else {k: v.detach() for k, v in wq.items()}
        p = leaf(wp, torch.float32) if side == "p" else {k: v.detach() for k, v in wp.items()}
        head.kl_divergence(q, p).sum().backward()
        assert wants == [(side == "q", side == "p")] * len(wq), (side, wants)
        assert all((q[k].grad is not None) == (side == "q") and (p[k].grad is not None) == (side == "p") for k in wq), side
    # no double backward
    p = leaf(wp, torch.float32)
    with pytest.raises(NotImplementedError):
        torch.autograd.grad(head.entropy(p).sum(), list(p.values()), create_graph=True)


def test_policies_have_the_reference_methods_and_state_dict_keys(emulated):
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "rl_gradient.pt"), weights_only=False)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), small_kwargs(), vpt_b200.PI_HEAD_KWARGS)
    assert [k for k, _, _ in fx["schema"]] == list(pol.state_dict())
    idm_fx = torch.load(os.path.join(ROOT, "tests", "golden", "idm.pt"), weights_only=False)
    from test_idm import SMALL_IDM

    idm = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs(**SMALL_IDM))
    assert [s[0] for s in idm_fx["small_schema"]] == list(idm.state_dict())
    for p, space in ((pol, "agent"), (idm, "idm")):
        assert isinstance(p.pi_head, _DictActionHead) and list(p.pi_head) == [n for n, _, _ in SPACES[space]]
        for name, shape, n in SPACES[space]:
            assert isinstance(p.pi_head[name], _CategoricalActionHead) and p.pi_head[name].output_shape == (*shape, n)
        pd = make_pd(space, B=2, T=3)
        assert torch.equal(p.pi_head.entropy(pd), getattr(p.pi_head, "entropy")(pd))
        ac = actions_for(space, B=2, T=3)
        assert torch.equal(p.logprob(ac, pd), p.pi_head.logprob(ac, pd))
        torch.manual_seed(4)
        a = p.sample(pd)
        torch.manual_seed(4)
        b = p.pi_head.sample(pd)
        assert all(torch.equal(a[k], b[k]) for k in a)
    pq, pp = make_pd("agent", B=2, T=3, seed=8), make_pd("agent", B=2, T=3, seed=9)
    kl = pol.get_kl_of_action_dists(pq, pp)
    old = sum((torch.exp(pq[k]) * (pq[k] - pp[k])).sum(-1, keepdim=True).sum(-2) for k in pq)  # the torch ops it replaced
    assert kl.shape == old.shape == (2, 3, 1) and torch.allclose(kl, old, rtol=1e-6, atol=1e-6)


def _rl_call(pol, sd, sd_ref, cfg, ent_coef=None, seed=0, B=2, T=8):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    first[1, 3] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    pd_ref, _ = ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, B))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, B))
    old, adv, returns = make_rl_batch(g, O.logprob(pd0, actions), B, T)
    tr = RLTrainer(pol)
    kw = dict(vf_coef=0.5, kl_coef=0.1) if ent_coef is None else dict(vf_coef=0.5, kl_coef=0.1, ent_coef=ent_coef)
    loss, _ = tr.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, **kw)
    return tr, loss, (img, first, actions, old, adv, returns, pd_ref)


def test_rl_entropy_bonus_is_the_exact_gradient(emulated, exact):
    """loss = L_pi + vf_coef L_v + kl_coef L_kl - ent_coef mean H(pi), against autograd through the oracle with the reference's entropy."""
    ent_coef = 0.3
    pol, sd, sd_ref, cfg = make_pair()
    norm = {k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM}
    tr, loss, (img, first, actions, old, adv, returns, pd_ref) = _rl_call(pol, sd, sd_ref, cfg, ent_coef)
    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}
    (pd, vpred, _), _ = O.agent_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    ent = ref_entropy(pd).mean()
    loss_o = rl_loss(pd, vpred, actions, old, adv, returns, pd_ref, norm, 0.5, 0.1, 0.2) - ent_coef * ent
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    assert abs(tr.stats["entropy"].item() - ent.item()) < 1e-5 * ent.item() and tr.stats["entropy"].dim() == 0
    n = 0
    for name, p in pol.named_parameters():
        g_o = leaf[name].grad
        if name.startswith("value_head.normalizer."):
            continue
        err = ((p.grad - g_o).norm() / g_o.norm().clamp(min=1e-12)).item()
        assert err < (5e-2 if name.startswith("net.img_process.cnn") else 1e-3), (name, err)
        n += 1
    assert n > 80
    # the bonus moves the heads' gradients: the same call without it differs
    pol2, sd2, sd_ref2, cfg2 = make_pair()
    _rl_call(pol2, sd2, sd_ref2, cfg2, 0.0)
    assert not torch.allclose(pol2.pi_head.buttons.linear_layer.weight.grad, pol.pi_head.buttons.linear_layer.weight.grad)


def test_rl_without_entropy_bonus_is_the_call_without_it(emulated, monkeypatch):
    """ent_coef = 0 runs the step of the trainer without the keyword, bit for bit (bf16 rounding on), and never the fused entry; the
    entropy statistic is still there, made when it is read, and equals the fused entry's of a call with the bonus."""
    fused = []
    monkeypatch.setattr(ops, "rl_head_bwd_ent", lambda *a, **k: fused.append(1) or emu_dist_ops.rl_head_bwd_ent(*a, **k))
    pol0, sd, sd_ref, cfg = make_pair()
    res = []
    for ent_coef in (None, 0.0, 0.02):
        pol = copy.deepcopy(pol0)
        tr, loss, _ = _rl_call(pol, sd, sd_ref, cfg, ent_coef)
        res.append((loss, {n: p.grad for n, p in pol.named_parameters()}, {k: getattr(pol.value_head.normalizer, k).clone() for k in NORM},
                    tr.stats))
        assert bool(fused) == bool(ent_coef)
    (l0, g0, n0, s0), (l1, g1, n1, s1), (l2, _, _, s2) = res
    assert torch.equal(l0, l1) and all(torch.equal(n0[k], n1[k]) for k in NORM)
    assert all((g0[n] is None and g1[n] is None) or torch.equal(g0[n], g1[n]) for n in g0)
    assert all(torch.equal(s0[k], s1[k]) for k in ("pi_loss", "vf_loss", "kl_ref", "clipfrac"))
    assert "entropy" in s0 and torch.equal(s0.get("entropy"), s0["entropy"]) and "entropy" in dict(s0.items())
    assert s1["entropy"].dim() == 0 and torch.equal(s0["entropy"], s1["entropy"])
    assert torch.allclose(s1["entropy"], s2["entropy"], rtol=1e-6, atol=0)
    with pytest.raises(KeyError):
        s1["nope"]


def test_rl_entropy_statistic_is_freed_by_the_next_call(emulated):
    """With ent_coef == 0 the unread entropy statistic holds the call's log-probs only until the trainer's next call starts."""
    pol, sd, sd_ref, cfg = make_pair()
    tr, _, args = _rl_call(pol, sd, sd_ref, cfg)
    first_stats = tr.stats
    assert "entropy" in first_stats and first_stats._lazy
    tr.loss_and_grad(args[0], args[1], pol.initial_state(2), *args[2:], vf_coef=0.5, kl_coef=0.1)
    assert not first_stats._lazy and "entropy" not in first_stats
    with pytest.raises(KeyError):
        first_stats["entropy"]
    assert tr.stats["entropy"].dim() == 0
