"""The head distribution kernels (csrc/head_dist.cuh) and the RL head backward with the entropy bonus (csrc/rl_bwd.cuh) on the GPU: against
float64 references with NaN-filled outputs between NaN guards and bit-identical reruns, at the RL / BC call shape (2048 rows of the
121- and 8641-wide agent heads), at an odd row count and on the IDM's factored layouts; `pi_head.entropy` in a 2x `loss.backward()` step
against the torch-op formula; `RLTrainer` with ent_coef = 0 against the call without the keyword."""
import copy

import pytest
import torch

import vpt_b200
from test_rl_training import make_pair, make_rl_batch
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.training import RLTrainer

pytestmark = pytest.mark.gpu
GUARD = 64
# (rows, groups, n): the agent's camera and buttons heads at the 2048-frame call, an odd row count, the IDM's buttons and camera heads
LAYOUTS = [(2048, 1, 121), (2048, 1, 8641), (333, 1, 8641), (1001, 1, 121), (512, 20, 2), (512, 2, 11)]


def _logp(rows, groups, n, g, masked=True):
    x = 3.0 * torch.randn(rows, groups, n, generator=g, dtype=torch.float64)
    if masked:
        x[torch.rand(x.shape, generator=g) < 0.2] = -100.0  # masked logits (policy.py `_heads`)
    return torch.log_softmax(x, -1).reshape(rows, groups * n).float()


def _rows_in(x, ld):
    """x [rows, width] as a device view with row stride ld, NaN in the columns past width and in guard rows around it."""
    rows, width = x.shape
    buf = torch.full((rows + 2, ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[1:rows + 1, :width] = x.cuda()
    return buf, buf[1:rows + 1, :width]


def _nan_out(*shape):
    buf = torch.full((shape[0] * (shape[1] if len(shape) > 1 else 1) + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    return buf, buf[GUARD:GUARD + buf.numel() - 2 * GUARD].view(*shape)


def _guards_intact(buf):
    return bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())


def _fwd(kind, lq, lp, groups, n, rows):
    buf, out = _nan_out(rows)
    if kind == "entropy":
        rc = nat.lib().vpt_head_entropy(lp.data_ptr(), lp.stride(0), groups, n, out.data_ptr(), rows, ops._stream())
    else:
        rc = nat.lib().vpt_head_kl(lq.data_ptr(), lq.stride(0), lp.data_ptr(), lp.stride(0), groups, n, out.data_ptr(), rows, ops._stream())
    nat.check(rc)
    torch.cuda.synchronize()
    assert _guards_intact(buf)
    return out.clone()


@pytest.mark.parametrize("rows,groups,n", LAYOUTS)
def test_forward_kernels_match_float64(rows, groups, n):
    g = torch.Generator().manual_seed(rows * 7 + n)
    width = groups * n
    lp32, lq32 = _logp(rows, groups, n, g), _logp(rows, groups, n, g)
    _, lp = _rows_in(lp32, width + 5)
    _, lq = _rows_in(lq32, width + 3)
    p64, q64 = lp32.double(), lq32.double()
    for kind, ref, terms in (("entropy", -(p64.exp() * p64).sum(-1), (p64.exp() * p64).abs().sum(-1)),
                             ("kl", (q64.exp() * (q64 - p64)).sum(-1), (q64.exp() * (q64.abs() + p64.abs())).sum(-1))):
        a, b = _fwd(kind, lq, lp, groups, n, rows), _fwd(kind, lq, lp, groups, n, rows)
        assert torch.isfinite(a).all() and torch.equal(a, b), kind
        err = ((a.double().cpu() - ref).abs() / (terms + 1e-30)).max().item()
        print(f"{kind} rows={rows} groups={groups} n={n}: worst error {err:.2e} of the sum of |terms|")
        assert err < 1e-5, (kind, err)
    # the tensor wrappers return the same bits
    assert torch.equal(ops.head_entropy(lp, groups), _fwd("entropy", lq, lp, groups, n, rows))
    assert torch.equal(ops.head_kl(lq, lp, groups), _fwd("kl", lq, lp, groups, n, rows))


@pytest.mark.parametrize("rows,groups,n", LAYOUTS)
def test_backward_kernels_match_float64_autograd(rows, groups, n):
    g = torch.Generator().manual_seed(rows * 5 + n)
    width = groups * n
    lp32, lq32 = _logp(rows, groups, n, g), _logp(rows, groups, n, g)
    up = torch.randn(rows, generator=g, dtype=torch.float64).float()
    _, lp = _rows_in(lp32, width + 1)
    _, lq = _rows_in(lq32, width + 7)
    gc = up.cuda()
    p64 = lp32.double().requires_grad_(True)
    q64 = lq32.double().requires_grad_(True)
    (-(p64.exp() * p64).sum(-1) * up.double()).sum().backward()
    dp_ent = p64.grad.clone()
    p64.grad = None
    ((q64.exp() * (q64 - p64)).sum(-1) * up.double()).sum().backward()
    ld = width + 4
    runs = []
    for _ in range(2):
        bufs = [torch.full((rows * ld + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda") for _ in range(3)]
        outs = [b[GUARD:GUARD + rows * ld].view(rows, ld) for b in bufs]
        nat.check(nat.lib().vpt_head_entropy_bwd(lp.data_ptr(), lp.stride(0), gc.data_ptr(), groups, n, outs[0].data_ptr(), ld, rows, ops._stream()))
        nat.check(nat.lib().vpt_head_kl_bwd(lq.data_ptr(), lq.stride(0), lp.data_ptr(), lp.stride(0), gc.data_ptr(), groups, n, outs[1].data_ptr(),
                                            ld, outs[2].data_ptr(), ld, rows, ops._stream()))
        torch.cuda.synchronize()
        for b, o in zip(bufs, outs):
            assert _guards_intact(b) and torch.isnan(o[:, width:]).all() and torch.isfinite(o[:, :width]).all()
        runs.append([o[:, :width].clone() for o in outs])
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    # errors relative to the size of the operands (lq - lp + 1 may cancel)
    P, Q, U = lp32.double(), lq32.double(), up.double().abs()[:, None]
    for name, got, ref, size in (("entropy dlogp", runs[0][0], dp_ent, U * P.exp() * (P.abs() + 1)),
                                 ("kl dlogq", runs[0][1], q64.grad, U * Q.exp() * (Q.abs() + P.abs() + 1)), ("kl dlogp", runs[0][2], p64.grad, U * Q.exp())):
        err = ((got.double().cpu() - ref).abs() / (size + 1e-30)).max().item()
        print(f"{name} rows={rows} groups={groups} n={n}: worst rel error {err:.2e}")
        assert err < 2e-6, (name, err)
    # one side of the KL: the other is not written
    dq, dp = ops.head_kl_bwd(lq, lp, gc, groups, want_q=False)
    assert dq is None and torch.equal(dp, runs[0][2])
    assert torch.equal(ops.head_entropy_bwd(lp, gc, groups), runs[0][0])


def _rl_entry(fused, logp, idx, c, logq, k, e, inv_temp, n, rows, col0=3, ld_out=None):
    ld_out = ld_out or col0 + n + 5
    out = torch.full((rows, ld_out), float("nan"), dtype=torch.bfloat16, device="cuda")
    kl = torch.full((rows,), float("nan"), device="cuda")
    ent = torch.full((rows,), float("nan"), device="cuda")
    q = 0 if logq is None else logq.data_ptr()
    ldq = 0 if logq is None else logq.stride(0)
    if fused:
        rc = nat.lib().vpt_rl_head_bwd_ent(logp.data_ptr(), logp.stride(0), q, ldq, idx.data_ptr(), c.data_ptr(), k, e, inv_temp, n, out.data_ptr(),
                                           ld_out, col0, kl.data_ptr(), ent.data_ptr(), 0, rows, ops._stream())
    else:
        rc = nat.lib().vpt_rl_head_bwd(logp.data_ptr(), logp.stride(0), q, ldq, idx.data_ptr(), c.data_ptr(), k, inv_temp, n, out.data_ptr(), ld_out,
                                       col0, kl.data_ptr(), 0, rows, ops._stream())
    nat.check(rc)
    torch.cuda.synchronize()
    assert torch.isnan(out[:, :col0].float()).all() and torch.isnan(out[:, col0 + n:].float()).all()
    return out, kl, ent


@pytest.mark.parametrize("rows,n", [(2048, 121), (2048, 8641), (333, 8641), (1001, 121)])
def test_fused_rl_entry(rows, n):
    g = torch.Generator().manual_seed(rows + n)
    lp32, lq32 = _logp(rows, 1, n, g), _logp(rows, 1, n, g)
    _, lp = _rows_in(lp32, n + 3)
    _, lq = _rows_in(lq32, n + 1)
    idx = torch.randint(0, n, (rows,), generator=g)
    c = (torch.randn(rows, generator=g, dtype=torch.float64) / rows).float()
    k, inv_temp, e = 0.1 / rows, 0.5, 0.3 / rows
    idx_c, c_c = idx.cuda(), c.cuda()
    for logq in (lq, None):
        base = _rl_entry(False, lp, idx_c, c_c, logq, k, 0.0, inv_temp, n, rows)
        zero = _rl_entry(True, lp, idx_c, c_c, logq, k, 0.0, inv_temp, n, rows)
        # ent_coef == 0: vpt_rl_head_bwd's bits, and the entropy of vpt_head_entropy
        assert torch.equal(zero[0].view(torch.int16), base[0].view(torch.int16)) and torch.equal(zero[1], base[1])
        assert torch.equal(zero[2], ops.head_entropy(lp))
        a, b = _rl_entry(True, lp, idx_c, c_c, logq, k, e, inv_temp, n, rows), _rl_entry(True, lp, idx_c, c_c, logq, k, e, inv_temp, n, rows)
        assert all(torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x, y.view(torch.int16) if y.dtype == torch.bfloat16 else y)
                   for x, y in zip(a, b))
        assert torch.equal(a[1], base[1]) and torch.equal(a[2], zero[2])
        p64 = lp32.double()
        p = p64.exp()
        H = -(p * p64).sum(-1, keepdim=True)
        ref = c.double()[:, None] * p
        ref[torch.arange(rows), idx] -= c.double()
        if logq is not None:
            ref = ref + k * (p - lq32.double().exp())
        ref = (ref + e * p * (p64 + H)) * inv_temp
        got = a[0][:, 3:3 + n].double().cpu()
        assert torch.isfinite(got).all()
        err = ((got - ref).abs() / (ref.abs() + 1e-3 * ref.abs().max())).max().item()
        print(f"rl_head_bwd_ent rows={rows} n={n} logq={'yes' if logq is not None else 'no'}: worst rel error {err:.2e}")
        assert err < 8e-3, err  # bf16 output: half an ulp is 2^-9 of the value
        h_err = ((zero[2].double().cpu() - H[:, 0]).abs() / (p * p64).abs().sum(-1)).max().item()
        assert h_err < 1e-5, h_err


def test_entropy_bonus_in_a_2x_loss_backward():
    """(nll - 0.01 * pi_head.entropy(pd).mean()).backward() on the 2x policy gives the gradients of the torch-op formula within fp32
    summation-order differences (the two upstream gradients of pd differ in their last bits before the bf16 head gradient)."""
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
    pol.set_autograd(True)
    g = torch.Generator().manual_seed(1)
    B, T = 2, 16
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    grads, ents = [], []
    for torch_ops in (False, True):
        pol.zero_grad(set_to_none=True)
        (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
        nll = -pol.logprob(actions, pd).mean()
        ent = sum(-(torch.exp(v) * v).sum(-1).sum(-1) for v in pd.values()) if torch_ops else pol.pi_head.entropy(pd)
        assert ent.shape == (B, T)
        (nll - 0.01 * ent.mean()).backward()
        ents.append(ent.detach())
        grads.append({n: p.grad.clone() for n, p in pol.named_parameters() if p.grad is not None})
    assert torch.allclose(ents[0], ents[1], rtol=1e-5, atol=0)
    assert set(grads[0]) == set(grads[1]) and len(grads[0]) > 100
    worst = 0.0
    for n, a in grads[0].items():
        b = grads[1][n]
        err = ((a - b).norm() / b.norm().clamp(min=1e-30)).item()
        worst = max(worst, err)
        assert err < 1e-3, (n, err)
    print(f"2x loss.backward with the entropy bonus: worst per-parameter rel-L2 difference to the torch-op formula {worst:.2e}")


def test_rl_trainer_entropy_bonus_on_the_gpu():
    """ent_coef = 0 gives the `.grad`, loss, statistics and normaliser of the call without the keyword bit for bit; ent_coef > 0 trains
    with the fused entry, and its entropy statistic is the one read lazily from the ent_coef = 0 call."""
    pol0, _, sd_ref, _ = make_pair()
    pol0 = pol0.cuda()
    ref = copy.deepcopy(pol0)
    ref.load_state_dict(sd_ref)
    g = torch.Generator().manual_seed(2)
    B, T = 2, 8
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    first[1, 3] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref.initial_state(B))
        (pd0, _, _), _ = pol0({"img": img}, first, pol0.initial_state(B))
    old, adv, returns = (x.cuda() for x in make_rl_batch(g, pol0.logprob(actions, pd0).cpu(), B, T))
    res = []
    for ent_coef in (None, 0.0, 0.01):
        pol = copy.deepcopy(pol0)
        tr = RLTrainer(pol)
        kw = {} if ent_coef is None else dict(ent_coef=ent_coef)
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1, **kw)
        res.append((loss, {n: p.grad for n, p in pol.named_parameters()}, [b.clone() for b in pol.value_head.normalizer.parameters()], tr.stats))
    (l0, g0, n0, s0), (l1, g1, n1, s1), (l2, g2, _, s2) = res
    assert torch.equal(l0, l1) and all(torch.equal(a, b) for a, b in zip(n0, n1))
    assert all((g0[n] is None and g1[n] is None) or torch.equal(g0[n], g1[n]) for n in g0)
    assert all(torch.equal(s0[k], s1[k]) for k in ("pi_loss", "vf_loss", "kl_ref", "clipfrac", "entropy"))
    assert s1["entropy"].dim() == 0 and s1["entropy"].is_cuda and torch.equal(s1["entropy"], s2["entropy"])
    assert torch.allclose(l2, l1 - 0.01 * s2["entropy"], rtol=1e-6, atol=0)
    n = "pi_head.camera.linear_layer.weight"
    assert torch.isfinite(g2[n]).all() and not torch.equal(g2[n], g1[n])
