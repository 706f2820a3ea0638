"""The differentiable forward on the H100: `vpt_log_softmax_bwd` against float64, and `loss.backward()` through the CUDA kernels against the
forced replica of its own tape, against BCTrainer, at the reference BC loop's one-frame shape, with both optimizers and at 3x width."""
import pytest
import torch
import torch.nn.functional as F

import vpt_b200
import vpt_oracle as O
from common import make_policy, perturb, small_kwargs
from test_autograd import bc_loss, custom_loss
from test_gpu_rl_training import no_tf32
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP
from video_pre_training_b200.training import BCTrainer

pytestmark = pytest.mark.gpu

GUARD = 0xFFFF  # bf16 NaN pattern of the guard columns


def _bf16_ulp(x):
    """One bf16 rounding step at |x| (8 significant bits)."""
    e = torch.floor(torch.log2(x.abs().clamp(min=1e-30)))
    return torch.exp2(e - 7)


@pytest.mark.parametrize("rows,n,groups", [(2048, 8641, 1), (2048, 121, 1), (512, 2, 20), (512, 11, 2)])
@pytest.mark.parametrize("masked", [False, True])
def test_log_softmax_bwd_matches_float64(rows, n, groups, masked):
    g = torch.Generator().manual_seed(rows + n + groups)
    width = n * groups
    logits = 3.0 * torch.randn(rows, groups, n, generator=g, dtype=torch.float64)
    mask = torch.rand(rows, width, generator=g) > 0.2 if masked else None
    if masked:
        logits = logits.masked_fill(~mask.view(rows, groups, n), -100.0)
    logp = torch.log_softmax(logits, -1).reshape(rows, width)
    up = torch.randn(rows, width, generator=g, dtype=torch.float64)
    scale = 0.5
    S = up.view(rows, groups, n).sum(-1, keepdim=True)
    ref = (scale * (up.view(rows, groups, n) - torch.exp(logp.view(rows, groups, n)) * S)).reshape(rows, width)
    if masked:
        ref = ref.masked_fill(~mask, 0.0)
    col0, ld = 24, width + 40
    outs = []
    for _ in range(2):
        out = torch.full((rows, ld), -1, dtype=torch.int16).view(torch.bfloat16).cuda()  # 0xFFFF
        ops.log_softmax_bwd(logp.float().cuda(), up.float().cuda(), scale, out, col0, groups, None if mask is None else mask.cuda())
        torch.cuda.synchronize()
        outs.append(out)
    o = outs[0].cpu()
    raw = o.view(torch.int16).to(torch.int32) & 0xFFFF
    assert (raw[:, :col0] == GUARD).all() and (raw[:, col0 + width:] == GUARD).all(), "guard columns written"
    got = o[:, col0:col0 + width].double()
    # fp32 inputs (logp, g rounded once each) and the bf16 store: one bf16 rounding of the result plus the fp32 noise of S * p
    tol = _bf16_ulp(ref) + 1e-6 * (S.abs().expand(rows, groups, n).reshape(rows, width) + up.abs()) * scale
    bad = (got - ref).abs() > tol
    assert not bad.any(), (bad.sum().item(), (got - ref).abs().max().item())
    if masked:
        assert (got[~mask] == 0).all()
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), "not bit-reproducible"


def test_log_softmax_bwd_one_hot_is_softmax_bwd():
    """The BC upstream gradient -onehot / N through the general kernel gives softmax_bwd's dlog to within one bf16 ulp."""
    g = torch.Generator().manual_seed(0)
    rows, n = 2048, 8641
    logp = torch.log_softmax(2.0 * torch.randn(rows, n, generator=g), -1).cuda()
    idx = torch.randint(0, n, (rows,), generator=g).cuda()
    up = torch.zeros(rows, n, device="cuda")
    up[torch.arange(rows, device="cuda"), idx] = -1.0 / rows
    a = torch.zeros(rows, n, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros_like(a)
    ops.log_softmax_bwd(logp, up, 0.5, a, 0)
    ops.softmax_bwd(logp, idx, 0.5 / rows, b, 0)
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    assert ((ia - ib).abs() <= 1).all()


def test_log_softmax_bwd_refuses_bad_arguments():
    lp = torch.zeros(4, 10, device="cuda")
    out = torch.zeros(4, 10, dtype=torch.bfloat16, device="cuda")
    lib = nat.lib()
    for args in ((lp.data_ptr(), 10, lp.data_ptr(), 10, None, 1, 10, 1.0, out.data_ptr(), 10, 1, 4, None),   # col0 + width > ld_out
                 (lp.data_ptr(), 5, lp.data_ptr(), 10, None, 1, 10, 1.0, out.data_ptr(), 10, 0, 4, None),    # ld_logp < width
                 (lp.data_ptr(), 10, lp.data_ptr(), 10, None, 0, 10, 1.0, out.data_ptr(), 10, 0, 4, None),   # no groups
                 (None, 10, lp.data_ptr(), 10, None, 1, 10, 1.0, out.data_ptr(), 10, 0, 4, None)):           # NULL logp
        with pytest.raises(nat.NativeError):
            nat.check(lib.vpt_log_softmax_bwd(*args), "vpt_log_softmax_bwd")
    with pytest.raises(ValueError):
        ops.log_softmax_bwd(lp, lp[:, :5].contiguous(), 1.0, out, 0)
    with pytest.raises(ValueError):
        ops.log_softmax_bwd(lp, lp, 1.0, out.float(), 0)
    with pytest.raises(ValueError):
        ops.log_softmax_bwd(lp, lp, 1.0, out, 0, groups=3)


def _grads(pol):
    return {n: None if p.grad is None else p.grad.clone() for n, p in pol.named_parameters()}


def _small_batch(B=2, T=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool)
    first[B - 1, T // 2] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    return img, first.cuda(), actions, g


def _forced_pd(leaf, cfg, tape, img, first, actions, B, t):
    from forced_replica_rl import forced_latent

    lat = forced_latent(leaf, cfg, tape, img, first, actions)
    pd = {}
    for name in ("camera", "buttons"):
        lin = f"pi_head.{name}.linear_layer"
        pd[name] = F.log_softmax(F.linear(lat, leaf[f"{lin}.weight"], leaf[f"{lin}.bias"]).float() / 2.0, dim=-1).reshape(B, t, 1, -1)
    vpred = F.linear(lat, leaf["value_head.linear.weight"], leaf["value_head.linear.bias"]).reshape(B, t, 1)
    return pd, vpred


def _vs_forced(pol, sd, cfg, img, first, actions, loss_fn):
    """Per-parameter rel-L2 of `loss.backward()`'s gradients against autograd through the forced replica of the call's own tape."""
    runner = pol._ag_runner
    B, t = img.shape[:2]
    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}
    with no_tf32():
        pd, vpred = _forced_pd(leaf, cfg, runner.last_tape, img, first, actions, B, t)
        lf = loss_fn(pd, vpred)
        lf.backward()
    worst = {}
    for n, p in pol.named_parameters():
        g_o = leaf[n].grad
        assert (p.grad is None) == (g_o is None), n
        if g_o is not None and g_o.any():
            worst[n] = ((p.grad - g_o).norm() / g_o.norm()).item()
    return lf.item(), worst


@pytest.mark.parametrize("which", ["bc", "custom"])
def test_small_autograd_matches_forced_replica(which):
    pol, sd, cfg = make_policy(small_kwargs())
    pol = pol.cuda().set_autograd(True)
    sd = {k: v.cuda() for k, v in sd.items()}
    img, first, actions, g = _small_batch()
    B, T = img.shape[:2]
    pd_ref = {k: torch.log_softmax(torch.randn(B, T, 1, n, generator=g), -1).cuda() for k, n in (("camera", 121), ("buttons", 8641))}
    target = (2.0 * torch.randn(B, T, generator=g)).cuda()
    if which == "bc":
        loss_fn = lambda pd, vpred: -O.logprob(pd, actions).mean()  # noqa: E731
    else:
        loss_fn = lambda pd, vpred: custom_loss(pd, vpred, actions, pd_ref, pol.denormalize, target)  # noqa: E731
    from video_pre_training_b200.policy import _autograd_runner

    _autograd_runner(pol).keep_tape = True
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    loss = loss_fn(pd, vpred)
    loss.backward()
    nat.device_check()
    lf, worst = _vs_forced(pol, sd, cfg, img, first, actions, loss_fn)
    print(f"{which}: autograd vs forced replica, worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4], "loss", loss.item(), lf)
    assert abs(loss.item() - lf) < 1e-3 * abs(lf)
    bad = {n: e for n, e in worst.items() if e > 3e-2}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


def test_autograd_bc_matches_bctrainer():
    """The same batch through BCTrainer and through loss.backward(): the same forward, dlog within one bf16 ulp."""
    pol, _, _ = make_policy(small_kwargs())
    pol = pol.cuda()
    img, first, actions, _ = _small_batch(seed=3)
    loss_t, _ = BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
    ref = _grads(pol)
    pol.zero_grad(set_to_none=True)
    (pd, _, _), _ = pol.set_autograd(True)({"img": img}, first, pol.initial_state(2))
    loss = bc_loss(pol, pd, actions)
    loss.backward()
    assert torch.equal(loss.detach(), loss_t), (loss.item(), loss_t.item())
    worst = {}
    for n, p in pol.named_parameters():
        assert (p.grad is None) == (ref[n] is None), n
        if ref[n] is not None and ref[n].any():
            worst[n] = ((p.grad - ref[n]).norm() / ref[n].norm()).item()
    print("autograd BC vs BCTrainer, worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4])
    assert max(worst.values()) < 1e-2


def _policy(width, **over):
    kw = vpt_b200.policy_kwargs(width, **over)
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    return pol.cuda(), kw


def test_reference_bc_loop_shape_at_2x():
    """behavioural_cloning.py:86-123 as written: B = 1, T = 1 per call, the state carried and detached, backward per sample; the 128-frame
    memory first filled by an inference chunk.  Finite gradients, and the last sample against the forced replica of its tape."""
    pol, kw = _policy("2x", n_recurrence_layers=4)
    cfg = O.Cfg(**kw)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    img0 = torch.randint(0, 256, (1, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    with torch.no_grad():
        _, state = pol({"img": img0}, torch.zeros(1, 128, dtype=torch.bool).cuda(), pol.initial_state(1))
    pol.set_autograd(True)
    from video_pre_training_b200.policy import _autograd_runner

    _autograd_runner(pol).keep_tape = True
    for i in range(8):
        obs = {"img": torch.randint(0, 256, (1, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()}
        action = {"camera": torch.randint(0, 121, (1, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (1, 1), generator=g).cuda()}
        if i == 7:
            pol.zero_grad(set_to_none=True)
            st_in = state
        pd, v, state = pol.get_output_for_observation(obs, state, torch.zeros(1, dtype=torch.bool))
        log_prob = pol.get_logprob_of_action(pd, action)
        state = [(m, (k.detach(), v_.detach())) for m, (k, v_) in state]
        (-log_prob / 8).backward()
    nat.device_check()
    for n, p in pol.named_parameters():
        assert n.startswith("value_head") == (p.grad is None), n
        if p.grad is not None:
            assert torch.isfinite(p.grad).all(), n
    img = obs["img"].unsqueeze(1)
    first = torch.zeros(1, 1, dtype=torch.bool).cuda()
    acts = {k: v.unsqueeze(1) for k, v in action.items()}
    del st_in
    lf, worst = _vs_forced(pol, {k: v.cuda() for k, v in sd.items()}, cfg, img, first, acts, lambda pd, vpred: -O.logprob(pd, acts).mean() / 8)
    print("2x B=1 T=1 vs forced replica, worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4])
    bad = {n: e for n, e in worst.items() if e > 3e-2}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]


@pytest.mark.parametrize("opt_kind", ["flat", "torch"])
def test_optimizers_step_on_autograd_gradients(opt_kind):
    pol, _, _ = make_policy(small_kwargs())
    pol = pol.cuda().set_autograd(True)
    img, first, actions, _ = _small_batch(seed=5)
    params = [p for n, p in pol.named_parameters() if p.requires_grad and not n.startswith("value_head")]
    opt = FlatAdamDP(params, lr=3e-4) if opt_kind == "flat" else torch.optim.Adam(params, lr=3e-4)
    losses = []
    for _ in range(4):
        opt.zero_grad()
        (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(2))
        loss = bc_loss(pol, pd, actions)
        loss.backward()
        if opt_kind == "flat":
            base = opt.flat_g.data_ptr()
            assert all(base <= p.grad.data_ptr() < base + opt.flat_g.numel() * 4 for p in params), ".grad no longer aliases the bucket"
        opt.step()
        losses.append(loss.item())
    print(opt_kind, "losses", losses)
    assert losses[-1] < losses[0]


def test_3x_short_clip_through_autograd():
    """Every backward kernel at production width through the new entry (cf. test_bc_step_at_3x_width_shapes)."""
    pol, _ = _policy("3x")
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(2)
    B, T = 2, 16
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    (bc_loss(pol, pd, actions) + 0.1 * (vpred ** 2).mean()).backward()
    nat.device_check()
    for n, p in pol.named_parameters():
        if n.startswith("value_head.normalizer."):
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.any(), n
