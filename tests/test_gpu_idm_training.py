"""IDM training step on the GPU: the three IDM backward kernels against float64 references, a SMALL_IDM step against the emulated CPU
step and its own forced replica, and the 4x IDM at full width (per parameter against the forced replica) and at 512 frames per call.

Bounds sit beside the worst value measured on an H100 80GB HBM3 (700 W)."""

import pytest
import torch

import emu_idm_ops
import emu_ops
import vpt_b200
from common import emulation
from test_idm_training import check_pattern, kind, make_batch, make_idm
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.training import IDMTrainer

pytestmark = pytest.mark.gpu
GUARD = 64


def _guarded(n, dev="cuda"):
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=torch.float32, device=dev)
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf, n):
    return torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all()


def _conv3d_bwd_raw(img, dy, C_):
    B, T, H, W, _ = img.shape
    bw, dW = _guarded(C_ * 15)
    bb, db = _guarded(C_)
    ws = torch.empty((nat.lib().vpt_conv3d_t5_bwd_workspace(B * T, H, W, C_),), dtype=torch.float32, device="cuda")
    nat.check(nat.lib().vpt_conv3d_t5_bwd(img.data_ptr(), dy.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), B, T, H, W, C_,
                                          torch.cuda.current_stream().cuda_stream), "vpt_conv3d_t5_bwd")
    torch.cuda.synchronize()
    assert _guards_intact(bw, C_ * 15) and _guards_intact(bb, C_)
    return dW.view(C_, 15).clone(), db.clone()


@pytest.mark.parametrize("C_", [64, 128])
@pytest.mark.parametrize("B,T", [(1, 1), (3, 3), (2, 8), (2, 128)])
def test_conv3d_t5_bwd_matches_float64(C_, B, T):
    """Time windows clipped at both ends, no leakage between the B sequences of a call, (2, 128) = 256 frames = two frame slabs per
    block; ReLU-masked dy whose ZP pad row / column holds non-zero values that must not contribute."""
    g = torch.Generator().manual_seed(C_ + T)
    H = W = 16
    img = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g)
    d = torch.randn(B * T, H, W, C_, generator=g) * (torch.rand(B * T, H, W, C_, generator=g) > 0.3)
    dy = emu_ops.to_zp(d).to(torch.bfloat16)
    ref_w, ref_b = emu_idm_ops.conv3d_t5_bwd(img, dy, C_)  # float64 autograd of the conv3d, per-sequence padding
    dy[:, -1] = 7.0  # non-zero ZP pad row / column: a kernel that summed over them would fail (the reference reads the interior only)
    dy[:, :, -1] = -5.0
    got_w, got_b = _conv3d_bwd_raw(img.cuda(), dy.cuda(), C_)
    again_w, again_b = _conv3d_bwd_raw(img.cuda(), dy.cuda(), C_)
    assert torch.equal(got_w, again_w) and torch.equal(got_b, again_b)
    ew = ((got_w.cpu() - ref_w).double().norm() / ref_w.double().norm()).item()
    eb = ((got_b.cpu() - ref_b).double().norm() / ref_b.double().norm()).item()
    assert ew < 1e-5 and eb < 1e-5, (ew, eb)  # fp32 sums of exact bf16 x u8 products


def _attn_ref(q, k, v, dO, B, t, heads):
    h = q.shape[-1]
    D = h // heads
    qq = q.double().reshape(B, t, heads, D).permute(0, 2, 1, 3).requires_grad_(True)
    kk = k.double().reshape(B, t, heads, D).permute(0, 2, 1, 3).requires_grad_(True)
    vv = v.double().reshape(B, t, heads, D).permute(0, 2, 1, 3).requires_grad_(True)
    o = torch.softmax(qq @ kk.transpose(-1, -2) / D, -1) @ vv
    gq, gk, gv = torch.autograd.grad(o, (qq, kk, vv), dO.double().reshape(B, t, heads, D).permute(0, 2, 1, 3))
    f = lambda x: x.permute(0, 2, 1, 3).reshape(B * t, h)
    return f(gq), f(gk), f(gv)


@pytest.mark.parametrize("t", [8, 100, 128])
@pytest.mark.parametrize("heads", [2, 32])
def test_unmasked_attention_bwd_matches_float64(t, heads):
    B = 4 if heads == 2 else 2
    h = heads * 128
    g = torch.Generator().manual_seed(t * heads)
    q = (torch.randn(B * t, h, generator=g) * 3).to(torch.bfloat16)
    k = (torch.randn(B, t, h, generator=g) * 3).to(torch.bfloat16)
    v = torch.randn(B, t, h, generator=g).to(torch.bfloat16)
    dO = torch.randn(B * t, h, generator=g).to(torch.bfloat16)
    ref = _attn_ref(q, k, v, dO, B, t, heads)
    qc, kc, vc, dc = q.cuda(), k.cuda(), v.cuda(), dO.cuda()
    ld = 3 * h + 16
    outs = []
    for _ in range(2):
        out = torch.full((B * t + 2, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
        assert ops.attention_bwd(qc, kc, vc, None, None, None, None, dc, out[1:B * t + 1], B, t, 0, heads, causal=False) is None
        torch.cuda.synchronize()
        assert torch.isnan(out[0]).all() and torch.isnan(out[-1]).all() and torch.isnan(out[1:-1, 3 * h:]).all()
        outs.append(out[1:-1, :3 * h].clone())
    assert torch.equal(outs[0], outs[1])
    for i, r in enumerate(ref):
        got = outs[0][:, i * h:(i + 1) * h].double().cpu()
        e = ((got - r).norm() / r.norm()).item()
        assert e < 1e-2, (i, e)  # bf16 output rounding (~3e-3) on fp32 arithmetic


def test_causal_attention_bwd_is_unchanged_around_the_unmasked_kernel():
    """The causal path returns the same bits before and after unmasked calls (no shared state between the two kernels)."""
    B, t, maxlen, heads = 2, 16, 32, 2
    h = heads * 128
    g = torch.Generator().manual_seed(0)
    q = torch.randn(B * t, h, generator=g).to(torch.bfloat16).cuda()
    kf = torch.randn(B, maxlen + t, h, generator=g).to(torch.bfloat16).cuda()
    vf = torch.randn(B, maxlen + t, h, generator=g).to(torch.bfloat16).cuda()
    R = torch.randn(B * t, 10 * heads, generator=g).cuda()
    b_nd = torch.randn(10, maxlen, generator=g).cuda()
    first = torch.zeros(B, t, dtype=torch.uint8, device="cuda")
    smask = torch.ones(B, maxlen, dtype=torch.uint8, device="cuda")
    dO = torch.randn(B * t, h, generator=g).to(torch.bfloat16).cuda()

    def causal():
        out = torch.zeros(B * t, 3 * h + 10 * heads, dtype=torch.bfloat16, device="cuda")
        db = ops.attention_bwd(q, kf, vf, R, b_nd, first, smask, dO, out, B, t, maxlen, heads)
        return out, db

    o1, d1 = causal()
    out = torch.zeros(B * t, 3 * h, dtype=torch.bfloat16, device="cuda")
    ops.attention_bwd(q, kf[:, maxlen:].contiguous(), vf[:, maxlen:].contiguous(), None, None, None, None, dO, out, B, t, 0, heads, causal=False)
    o2, d2 = causal()
    assert torch.equal(o1, o2) and torch.equal(d1, d2)


@pytest.mark.parametrize("groups,n", [(20, 2), (2, 11)])
def test_grouped_head_bwd_matches_float64(groups, n):
    rows = 1000
    g = torch.Generator().manual_seed(groups)
    logits = torch.randn(rows, groups, n, generator=g, dtype=torch.float64) * 2
    logp = torch.log_softmax(logits, -1)
    idx = torch.randint(0, n, (rows, groups), generator=g)
    scale = 1.0 / 777
    ref = (torch.exp(logp) - torch.nn.functional.one_hot(idx, n).double()) * scale
    ref_lp = logp.gather(-1, idx[..., None]).squeeze(-1).sum(-1)
    c0 = 5
    out = torch.full((rows, c0 + groups * n + 3), float("nan"), dtype=torch.bfloat16, device="cuda")
    lp = ops.softmax_nll_bwd_grouped(logp.float().cuda(), idx.cuda(), scale, out, c0)
    lp2 = ops.softmax_nll_bwd_grouped(logp.float().cuda(), idx.cuda(), scale, out, c0, lp=lp.clone())
    o = out.cpu()
    assert torch.isnan(o[:, :c0]).all() and torch.isnan(o[:, c0 + groups * n:]).all()
    got = o[:, c0:c0 + groups * n].double().reshape(rows, groups, n)
    assert (got - ref).abs().max().item() <= 2 ** -8 * ref.abs().max().item()  # one bf16 rounding
    assert torch.allclose(lp.double().cpu(), ref_lp, rtol=1e-5, atol=1e-5)
    assert torch.allclose(lp2.double().cpu(), 2 * ref_lp, rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------------------
# whole steps
# ---------------------------------------------------------------------------------------------------------------------------------
def _grads(pol):
    return {n: None if p.grad is None else p.grad.detach().clone() for n, p in pol.named_parameters()}


def _step(pol, tr, img, first, actions, dev):
    for p in pol.parameters():
        p.grad = None
    B = img.shape[0]
    loss, _ = tr.loss_and_grad(img.to(dev), first.to(dev), pol.initial_state(B), {k: v.to(dev) for k, v in actions.items()})
    return loss.item(), _grads(pol)


def _vs_forced(pol, sd_dev, cfg, tr, img, actions, bound, temperature=2.0):
    from forced_replica_idm import forced_loss_idm

    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd_dev.items()}
    lf = forced_loss_idm(leaf, cfg, tr.last_tape, img, actions, temperature)
    lf.backward()
    worst = {}
    for n, p in pol.named_parameters():
        check_pattern(n, p.grad)
        if kind(n) != "dense":
            continue
        worst[n] = ((p.grad - leaf[n].grad).norm() / leaf[n].grad.norm()).item()
    print("forced replica: worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4])
    bad = {n: e for n, e in worst.items() if e > bound}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]
    return lf.item()


def test_small_idm_step_gpu():
    pol, sd, cfg = make_idm()
    img, first, actions = make_batch(torch.Generator().manual_seed(0))
    # emulated CPU step
    with emulation():
        from video_pre_training_b200 import ops as o_
        saved = {n: getattr(o_, n) for n in ("conv3d_t5_bwd", "softmax_nll_bwd_grouped")}
        for n in saved:
            setattr(o_, n, getattr(emu_idm_ops, n))
        try:
            loss_c, g_cpu = _step(pol, IDMTrainer(pol), img, first, actions, "cpu")
        finally:
            for n, f in saved.items():
                setattr(o_, n, f)
    pol = pol.cuda()
    tr = IDMTrainer(pol)
    tr.keep_tape = True
    loss_g, g1 = _step(pol, tr, img, first, actions, "cuda")
    nat.device_check()
    lf = _vs_forced(pol, {k: v.cuda() for k, v in sd.items()}, cfg, tr, img.cuda(), {k: v.cuda() for k, v in actions.items()}, 3e-2)  # measured worst 1.47e-2
    assert abs(loss_g - lf) < 1e-4 * abs(lf)
    assert abs(loss_g - loss_c) < 1e-2 * abs(loss_c)
    for n, g in g1.items():
        check_pattern(n, g)
        if kind(n) == "dense":
            cos = (g.cpu() * g_cpu[n]).sum() / (g.cpu().norm() * g_cpu[n].norm())
            assert cos > 0.9, (n, cos.item())
    _, g2 = _step(pol, tr, img, first, actions, "cuda")
    assert all((g1[n] is None and g2[n] is None) or torch.equal(g1[n], g2[n]) for n in g1), "IDM step not bit-reproducible"


def test_small_idm_loss_falls_with_adam():
    from video_pre_training_b200.parallel import FlatAdamDP

    pol, _, _ = make_idm()
    pol = pol.cuda()
    tr = IDMTrainer(pol)
    img, first, actions = make_batch(torch.Generator().manual_seed(1))
    img, first, actions = img.cuda(), first.cuda(), {k: v.cuda() for k, v in actions.items()}
    opt = FlatAdamDP(IDMTrainer.optimizer_params(pol), lr=3e-4)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(2), actions)
        losses.append(loss.item())
        opt.step()
    print("losses", losses)
    assert losses[-1] < 0.9 * losses[0], losses


def test_idm_4x_full_width_step_matches_forced_replica():
    """The released 4x IDM (idm_net_kwargs()), B = 1, T = 32, per parameter against the forced fp32 replica of its own tape."""
    torch.manual_seed(0)
    kw = vpt_b200.idm_net_kwargs(timesteps=32, attention_memory_size=32)  # mask "none": memory size == timesteps (no KV memory)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), kw).cuda()
    import vpt_oracle as O

    cfg = O.Cfg(conv3d=True, **{k: v for k, v in kw.items() if k != "conv3d_params"})
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    img, first, actions = make_batch(torch.Generator().manual_seed(2), B=1, T=32, hw=128)
    tr = IDMTrainer(pol)
    tr.keep_tape = True
    torch.cuda.reset_peak_memory_stats()
    _step(pol, tr, img, first, actions, "cuda")
    _vs_forced(pol, sd, cfg, tr, img.cuda(), {k: v.cuda() for k, v in actions.items()}, 5e-2)  # measured worst 1.48e-2 (conv3d weight)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"4x B=1 T=32 step + fp32 forced replica: peak {peak:.1f} GiB")
    assert peak < 32  # measured 18.4 GiB


def test_idm_4x_512_frame_step_equals_mean_of_single_sequences():
    """B = 4, T = 128 (512 frames: stack 0's full-resolution tensor is [512, 129, 129, 256], more than 2^31 elements) against the mean of
    four single-sequence steps; IDM sequences are independent, so only the fp32 summation order differs."""
    torch.manual_seed(0)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()
    tr = IDMTrainer(pol)
    img, first, actions = make_batch(torch.Generator().manual_seed(3), B=4, T=128, hw=128)
    img, first, actions = img.cuda(), first.cuda(), {k: v.cuda() for k, v in actions.items()}
    torch.cuda.reset_peak_memory_stats()
    loss4, g4 = _step(pol, tr, img, first, actions, "cuda")
    print(f"4x B=4 T=128 step: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    nat.device_check()
    mean, losses = {}, []
    for b in range(4):
        lb, gb = _step(pol, tr, img[b:b + 1], first[b:b + 1], {k: v[b:b + 1] for k, v in actions.items()}, "cuda")
        losses.append(lb)
        for n, g in gb.items():
            if g is not None:
                mean[n] = g / 4 if n not in mean else mean[n] + g / 4
    assert abs(loss4 - sum(losses) / 4) < 1e-5 * abs(loss4)
    worst = {}
    for n, g in g4.items():
        check_pattern(n, g)
        if kind(n) == "dense":
            worst[n] = ((g - mean[n]).norm() / mean[n].norm()).item()
    print("512 frames vs 4 x 128: worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4])
    bad = {n: e for n, e in worst.items() if e > 5e-3}  # measured worst 1.19e-3 (conv3d weight)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:8]
