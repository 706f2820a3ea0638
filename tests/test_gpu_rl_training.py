"""RL fine-tuning step on the GPU: the RL kernels (csrc/rl_bwd.cuh) against float64 references between NaN guard bands, a small RL step
against the emulated CPU step and the forced replica of its own tape, the 2x-width step per parameter against the forced replica, and a
few Adam steps on a fixed batch.

Bounds sit beside the worst value measured on an H100 80GB HBM3 at a 400 W power limit."""
import contextlib

import pytest
import torch

import emu_rl_ops
import vpt_b200
import vpt_oracle as O
from common import emulation, perturb
from test_rl_training import NORM, make_pair, make_rl_batch, ref_pd, rl_vs_forced
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.training import RLTrainer

pytestmark = pytest.mark.gpu
RL_OPS = ("ppo_coef", "rl_head_bwd", "ewma_sums", "value_bwd")


def _logp(rows, n, g, scale=3.0):
    return torch.log_softmax(torch.randn(rows, n, generator=g, dtype=torch.float64) * scale, -1)


def _mixed_rows(rows, g):
    """old_logprob / advantages with rows clipped on both sides and unclipped ones, none within 1e-3 of a boundary of clip = 0.2."""
    lp = -torch.rand(rows, generator=g, dtype=torch.float64) * 20
    ratio = torch.exp((torch.rand(rows, generator=g, dtype=torch.float64) - 0.5) * 1.4)
    ratio = torch.where((ratio - 1.2).abs() < 1e-3, ratio + 3e-3, ratio)
    ratio = torch.where((ratio - 0.8).abs() < 1e-3, ratio + 3e-3, ratio)
    adv = torch.randn(rows, generator=g, dtype=torch.float64)
    return lp, lp - torch.log(ratio), adv


def _ppo_ref(lp, old, adv, clip, rows):
    ratio = torch.exp(lp - old)
    clipped = ((adv > 0) & (ratio > 1 + clip)) | ((adv < 0) & (ratio < 1 - clip))
    c = torch.where(clipped, 0.0, ratio * adv / rows)
    return c, -torch.minimum(ratio * adv, ratio.clamp(1 - clip, 1 + clip) * adv), clipped.double()


@pytest.mark.parametrize("rows", [37, 2048])
def test_ppo_coef_matches_float64(rows):
    g = torch.Generator().manual_seed(rows)
    lp, old, adv = _mixed_rows(rows, g)
    outs = [ops.ppo_coef(lp.float().cuda(), old.float().cuda(), adv.float().cuda(), 0.2) for _ in range(2)]
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    c_ref, l_ref, f_ref = _ppo_ref(lp.float().double(), old.float().double(), adv.float().double(), 0.2, rows)
    c, l, f = (x.double().cpu() for x in outs[0])
    assert 0 < f_ref.sum() < rows and torch.equal(f, f_ref)
    err_c = ((c - c_ref).abs() / c_ref.abs().clamp(min=1e-30)).max().item()
    err_l = ((l - l_ref).abs() / l_ref.abs().clamp(min=1e-30)).max().item()
    print(f"ppo_coef rows={rows}: worst rel err c {err_c:.2e}, loss {err_l:.2e}")
    assert err_c < 5e-7 and err_l < 5e-7  # fp32 exp of an fp32 difference: measured worst 1.37e-7


@pytest.mark.parametrize("rows", [5, 2048])
@pytest.mark.parametrize("n", [121, 8641])
@pytest.mark.parametrize("with_ref", [True, False])
def test_rl_head_bwd_matches_float64(rows, n, with_ref):
    g = torch.Generator().manual_seed(rows + n + with_ref)
    logp = _logp(rows, n, g)
    logq = _logp(rows, n, g) if with_ref else None
    idx = torch.randint(0, n, (rows,), generator=g)
    c = torch.randn(rows, generator=g, dtype=torch.float64) / rows
    c[::3] = 0.0  # clipped rows
    k, inv_t = 0.1 / rows, 0.5
    p = torch.exp(logp.float().double())
    ref = c[:, None].float().double() * (p - torch.nn.functional.one_hot(idx, n).double())
    if with_ref:
        q = torch.exp(logq.float().double())
        ref = ref + k * (p - q)
        kl_ref = (q * (logq.float().double() - logp.float().double())).sum(-1)
    ref = ref * inv_t
    c0, G = 7, 16
    outs = []
    for _ in range(2):
        buf = torch.full((rows + 2, c0 + n + G), float("nan"), dtype=torch.bfloat16, device="cuda")
        prior = torch.full((rows,), 0.25, device="cuda")
        kl = ops.rl_head_bwd(logp.float().cuda(), idx.cuda(), c.float().cuda(), None if logq is None else logq.float().cuda(), k, inv_t,
                             buf[1:rows + 1], c0, prior)
        torch.cuda.synchronize()
        b = buf.cpu()
        assert torch.isnan(b[0]).all() and torch.isnan(b[-1]).all() and torch.isnan(b[:, :c0]).all() and torch.isnan(b[:, c0 + n:]).all()
        outs.append((b[1:-1, c0:c0 + n].clone(), kl.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    got, kl = outs[0][0].double(), outs[0][1].double() - 0.25
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    print(f"rl_head_bwd rows={rows} n={n} ref={with_ref}: max err / max |ref| {err:.2e}")
    assert err <= 2 ** -8  # one bf16 rounding: measured worst 2.68e-3
    if with_ref:
        e_kl = ((kl - kl_ref).abs().max() / kl_ref.abs().max()).item()
        print(f"  kl: max err / max kl {e_kl:.2e}")
        assert e_kl < 1e-6  # measured worst 3.16e-7 (n = 8641, 2048 rows)
    else:
        assert not kl.any()


@pytest.mark.parametrize("rows", [3, 2048])
def test_value_bwd_matches_float64(rows):
    g = torch.Generator().manual_seed(rows)
    ret = (5.0 + 3.0 * torch.randn(rows, generator=g)).float()
    vpred = torch.randn(rows, generator=g).float()
    start = (torch.tensor([0.7]), torch.tensor([2.5]), torch.tensor(0.3))
    ld, col = 24, 17
    results = []
    for _ in range(2):
        nz = [t.clone().cuda() for t in start]
        buf = torch.full((rows + 2, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
        sums = ops.ewma_sums(ret.cuda())
        sq = ops.value_bwd(vpred.cuda(), ret.cuda(), sums, rows, *nz, 0.99999, 0.37, buf[1:rows + 1], col)
        torch.cuda.synchronize()
        b = buf.cpu()
        assert torch.isnan(b[0]).all() and torch.isnan(b[-1]).all() and torch.isnan(b[:, :col]).all() and torch.isnan(b[:, col + 1:]).all()
        results.append((sums.cpu(), b[1:-1, col].clone(), sq.cpu(), [t.cpu() for t in nz]))
    a, b_ = results
    assert torch.equal(a[0], b_[0]) and torch.equal(a[1], b_[1]) and torch.equal(a[2], b_[2]) and all(torch.equal(x, y) for x, y in zip(a[3], b_[3]))
    r = ret.double()
    assert torch.allclose(a[0], torch.stack([r.sum(), (r * r).sum()]), rtol=1e-12, atol=0)
    w = 0.99999
    rm = start[0].double() * w + r.mean() * (1 - w)
    rsq = start[1].double() * w + (r * r).mean() * (1 - w)
    deb = start[2].double() * w + (1 - w)
    for got, want in zip(a[3], (rm, rsq, deb)):
        assert abs(got.double().item() - want.item()) <= 1e-6 * abs(want.item())
    mean = rm / deb
    var = (rsq / deb - mean ** 2).clamp(min=1e-2)
    d = vpred.double() - (r - mean) / var.sqrt()
    e_g = ((a[1].double() - 0.37 * d).abs().max() / (0.37 * d).abs().max()).item()
    e_sq = ((a[2].double() - d * d).abs().max() / (d * d).max()).item()
    print(f"value_bwd rows={rows}: dvpred {e_g:.2e}, sq err {e_sq:.2e}")
    assert e_g <= 2 ** -8 and e_sq < 1e-6  # one bf16 rounding (measured worst 2.90e-3); fp32 (measured worst 2.73e-7)


def test_rl_ops_refuse_bad_operands():
    rows, n = 8, 121
    logp = torch.log_softmax(torch.randn(rows, n), -1).cuda()
    c = torch.zeros(rows, device="cuda")
    out = torch.zeros(rows, n + 8, dtype=torch.bfloat16, device="cuda")
    idx = torch.zeros(rows, dtype=torch.int64, device="cuda")
    ops.rl_head_bwd(logp, idx, c, None, 0.0, 1.0, out, 0)
    for bad in (idx + n, idx - 1):
        with pytest.raises(ValueError):
            ops.rl_head_bwd(logp, bad, c, None, 0.0, 1.0, out, 0)
    with pytest.raises(ValueError):
        ops.rl_head_bwd(logp.double(), idx, c, None, 0.0, 1.0, out, 0)
    with pytest.raises(ValueError):
        ops.rl_head_bwd(logp.t().contiguous().t(), idx, c, None, 0.0, 1.0, out, 0)  # column stride != 1
    with pytest.raises(ValueError):
        ops.rl_head_bwd(logp, idx, c, logp[:, :100], 0.0, 1.0, out, 0)
    with pytest.raises(ValueError):
        ops.rl_head_bwd(logp, idx, c, None, 0.0, 1.0, out, 10)  # past the buffer's columns
    with pytest.raises(ValueError):
        ops.rl_head_bwd(logp, idx.int(), c, None, 0.0, 1.0, out, 0)
    with pytest.raises(ValueError):
        ops.ppo_coef(c, c[:4], c, 0.2)
    with pytest.raises(ValueError):
        ops.ppo_coef(c, c, c.double(), 0.2)
    nz = [torch.zeros(1, device="cuda") for _ in range(3)]
    with pytest.raises(ValueError):
        ops.value_bwd(c, c, torch.zeros(2, device="cuda"), rows, *nz, 0.99999, 1.0, out, n)  # fp32 sums
    with pytest.raises(ValueError):
        ops.value_bwd(c, c, torch.zeros(2, dtype=torch.float64, device="cuda"), rows, *nz, 0.99999, 1.0, out, n + 8)  # column out of range
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------------------
# whole steps
# ---------------------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def no_tf32():
    """The forced replica's fp32 layers in full fp32 (cuDNN would otherwise run its convolutions in TF32)."""
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32


def _grads(pol):
    return {n: None if p.grad is None else p.grad.detach().clone() for n, p in pol.named_parameters()}


def _batch(sd, sd_ref, cfg, B, T, hw, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (B, T, hw, hw, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    first[B - 1, T // 2] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, B))
    old, adv, returns = make_rl_batch(g, O.logprob(pd0, actions), B, T)
    pd_ref, _ = ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, B))
    return img, first, actions, old, adv, returns, pd_ref


def _rl_step(pol, tr, batch, dev, vf=0.5, kl=0.1):
    img, first, actions, old, adv, returns, pd_ref = batch
    for p in pol.parameters():
        p.grad = None
    B = img.shape[0]
    to = lambda x: x.to(dev)
    loss, _ = tr.loss_and_grad(to(img), to(first), pol.initial_state(B), {k: to(v) for k, v in actions.items()}, to(old), to(adv), to(returns),
                               {k: to(v) for k, v in pd_ref.items()}, vf_coef=vf, kl_coef=kl)
    return loss.item(), _grads(pol)


def test_small_rl_step_gpu():
    pol, sd, sd_ref, cfg = make_pair()
    batch = _batch(sd, sd_ref, cfg, 2, 8, 32, 0)
    norm0 = {k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM}
    with emulation():
        saved = {n: getattr(ops, n) for n in RL_OPS}
        for n in RL_OPS:
            setattr(ops, n, getattr(emu_rl_ops, n))
        try:
            loss_c, g_cpu = _rl_step(pol, RLTrainer(pol), batch, "cpu")
        finally:
            for n, f in saved.items():
                setattr(ops, n, f)
    norm_cpu = {k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM}
    with torch.no_grad():
        for k in NORM:
            getattr(pol.value_head.normalizer, k).copy_(norm0[k])
    pol = pol.cuda()
    tr = RLTrainer(pol)
    tr.keep_tape = True
    loss_g, g1 = _rl_step(pol, tr, batch, "cuda")
    nat.device_check()
    for k in NORM:
        assert torch.allclose(getattr(pol.value_head.normalizer, k).cpu(), norm_cpu[k], rtol=1e-6, atol=0), k
    cuda = lambda x: x.cuda()
    img, first, actions, old, adv, returns, pd_ref = batch
    with no_tf32():
        lf, worst = rl_vs_forced(pol, {k: v.cuda() for k, v in sd.items()}, cfg, tr, cuda(img), cuda(first), {k: cuda(v) for k, v in actions.items()},
                                 cuda(old), cuda(adv), cuda(returns), {k: cuda(v) for k, v in pd_ref.items()},
                                 {k: cuda(v) for k, v in norm0.items()}, 0.5, 0.1)
    print("small RL step vs forced replica: worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4], "loss", loss_g, lf, loss_c)
    assert abs(loss_g - lf) < 1e-3 * abs(lf) and abs(loss_g - loss_c) < 1e-2 * abs(loss_c)
    bad = {n: e for n, e in worst.items() if e > 3e-2}  # measured worst 1.33e-2
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]
    for n, g in g1.items():
        if g is None:
            assert g_cpu[n] is None, n
            continue
        cos = (g.cpu() * g_cpu[n]).sum() / (g.cpu().norm() * g_cpu[n].norm())
        assert cos > 0.9, (n, cos.item())
    assert g1["value_head.linear.weight"].abs().sum() > 0
    with torch.no_grad():
        for k in NORM:
            getattr(pol.value_head.normalizer, k).copy_(norm0[k])
    _, g2 = _rl_step(pol, tr, batch, "cuda")
    assert all((g1[n] is None and g2[n] is None) or torch.equal(g1[n], g2[n]) for n in g1), "RL step not bit-reproducible"


def test_rl_2x_step_matches_forced_replica():
    """The 2x policy (the width of the released RL models) with perturbed weights, B = 2, T = 64, an untaped chunk first so that the
    taped one carries state, per parameter against the forced fp32 replica of its own tape."""
    kw = vpt_b200.policy_kwargs("2x", n_recurrence_layers=4)
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    ref = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
    ref.load_state_dict(pol.state_dict())
    perturb(ref, seed=7)
    pol, ref = pol.cuda(), ref.cuda()
    cfg = O.Cfg(**kw)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    B, T = 2, 64
    g = torch.Generator().manual_seed(1)
    mk = lambda: (torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda(), torch.zeros(B, T, dtype=torch.bool).cuda())
    img0, first0 = mk()
    with torch.no_grad():
        _, st = pol({"img": img0}, first0, pol.initial_state(B))
        _, st_r = ref({"img": img0}, first0, ref.initial_state(B))
    img, first = mk()
    first[1, 20] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, st_r)
        (pd0, _, _), _ = pol({"img": img}, first, st)
    old, adv, returns = make_rl_batch(g, pol.logprob(actions, pd0).reshape(B, T).float().cpu(), B, T)
    old, adv, returns = old.cuda(), adv.cuda(), returns.cuda()
    norm0 = {k: getattr(pol.value_head.normalizer, k).detach().clone() for k in NORM}
    tr = RLTrainer(pol)
    tr.keep_tape = True
    torch.cuda.reset_peak_memory_stats()
    loss, _ = tr.loss_and_grad(img, first, st, actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)
    nat.device_check()
    del ref
    with no_tf32():
        lf, worst = rl_vs_forced(pol, {k: v.cuda() for k, v in sd.items()}, cfg, tr, img, first, actions, old, adv, returns, pd_ref, norm0, 0.5, 0.1)
    print("2x RL step vs forced replica: worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4], "loss", loss.item(), lf,
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    assert abs(loss.item() - lf) < 1e-3 * abs(lf)
    bad = {n: e for n, e in worst.items() if e > 5e-2}  # measured worst 1.41e-2; peak memory 17.6 GiB
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


def test_small_rl_adam_steps_move_the_policy():
    """A > 0 on a fixed batch: under Adam the chosen actions' log-prob rises, the KL to a reference equal to the starting weights stays
    small, and the value loss falls."""
    from video_pre_training_b200.parallel import FlatAdamDP

    pol, _, _, _ = make_pair()
    pol = pol.cuda()
    g = torch.Generator().manual_seed(9)
    B, T = 2, 8
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    with torch.no_grad():
        (pd0, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
    pd_ref = {k: v.clone() for k, v in pd0.items()}  # the reference policy: the starting weights
    old = pol.logprob(actions, pd0).reshape(B, T).float()
    adv = torch.ones(B, T, device="cuda")
    returns = (2.0 + torch.randn(B, T, generator=g)).cuda()
    tr = RLTrainer(pol)
    opt = FlatAdamDP([p for p in pol.parameters() if p.requires_grad], lr=1e-5)
    lps, kls, vfs = [], [], []
    for _ in range(6):
        opt.zero_grad()
        tr.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)
        kls.append(tr.stats["kl_ref"].item())
        vfs.append(tr.stats["vf_loss"].item())
        opt.step()
        with torch.no_grad():
            (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
        lps.append((pol.logprob(actions, pd).reshape(B, T) - old).mean().item())
    print("mean lp - old", lps, "kl", kls, "vf", vfs)
    # measured: mean lp - old 0.058 -> 0.318, largest KL 0.0196, value loss 1.50 -> 0.47
    assert lps[-1] > lps[0] > 0 and max(kls) < 0.05 and vfs[-1] < vfs[0]
