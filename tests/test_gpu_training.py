"""BC step on the GPU (SURVEY section 8 row a20): every backward kernel against the test-only emulation of the same op, and the
whole step (forward with tape + hand-written backward through the C ABI) against the emulated step and the oracle's autograd."""
import pytest
import torch

import emu_ops as E
import vpt_b200
import vpt_oracle as O
from common import emulation, make_policy, small_kwargs
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP
from video_pre_training_b200.training import BCTrainer, RLTrainer

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp(min=1e-20)).item()


def zp_rand(F_, H, W, C, g, scale=1.0, relu=False):
    x = torch.randn(F_, H, W, C, generator=g) * scale
    if relu:
        x = x.relu()
    return E.to_zp(x.to(BF16))


def test_relu_mask_and_residual_add():
    g = torch.Generator().manual_seed(0)
    d, o = zp_rand(3, 8, 8, 64, g), zp_rand(3, 8, 8, 64, g, relu=True)
    assert torch.equal(ops.relu_mask(d.to(DEV), o.to(DEV)).cpu(), E.relu_mask(d, o))
    a, b = zp_rand(3, 8, 8, 64, g), zp_rand(3, 8, 8, 64, g)
    s, mr = ops.add_zp(a.to(DEV), b.to(DEV), 8, 8)
    s_e, mr_e = E.add_zp(a, b, 8, 8)
    assert torch.equal(s.cpu(), s_e) and torch.allclose(mr.cpu(), mr_e, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("M,N,R,shifts", [
    (64, 64, 162, [(ky - 1) * 9 + (kx - 1) for ky in range(3) for kx in range(3)]),   # conv taps, tiny
    (192, 192, 2 * 65 * 65, [(ky - 1) * 65 + (kx - 1) for ky in range(3) for kx in range(3)]),  # 3x stack-0 shape, K split
    (128, 64, 5 * 33 * 33, [(ky - 1) * 33 + (kx - 1) for ky in range(3) for kx in range(3)]),
    (256, 1024, 2048, [0]),                                                             # linear
    (8768, 256, 300, [0]),                                                              # heads (many M tiles, K tail)
    (792, 256, 96, [0]),                                 # q|k|v|r concat (M not a multiple of 64)
    (384, 384, 3 * 33 * 33, [(ky - 1) * 33 + (kx - 1) for ky in range(3) for kx in range(3)]),  # 3x stack-1 shape: 3 m tiles x 2 n tiles
    (64, 128, 700, [0, 5, 6, 100]),                      # scattered tap shifts
    (256, 320, 1000, [-1, 0, 1]),                        # N tiles 128 + 128 + 64, taps with shifts -1 / 0 / 1
])
def test_wgrad_matches_emulation(M, N, R, shifts):
    g = torch.Generator().manual_seed(1)
    a = torch.randn(R, M, generator=g).to(BF16)
    b = torch.randn(R, N, generator=g).to(BF16)
    ref = E.wgrad(a, b, shifts)
    out = ops.wgrad(a.to(DEV), b.to(DEV), shifts)
    nat.device_check()
    assert out.shape == ref.shape and out.dtype == torch.float32
    assert rel(out, ref) < 1e-5 and (out.cpu() - ref).abs().max() < 1e-3 * ref.abs().max()
    # strided operands (a column slice of a wider buffer)
    wide = torch.randn(R, M + 64, generator=g).to(BF16)
    out2 = ops.wgrad(wide.to(DEV)[:, 64:], b.to(DEV), shifts)
    assert rel(out2, E.wgrad(wide[:, 64:], b, shifts)) < 1e-5
    try:  # every value of the kernel-choice knob gives the same sums (one weight-gradient kernel in this build)
        nat.lib().vpt_set_wgrad_mode(0)
        out0 = ops.wgrad(a.to(DEV), b.to(DEV), shifts)
        nat.device_check()
    finally:
        nat.lib().vpt_set_wgrad_mode(1)
    assert rel(out0, ref) < 1e-5


@pytest.mark.parametrize("rows,C,rpg,zp", [(2 * 81, 64, 81, (8, 8, 64)), (40, 256, 1, None), (6, 5 * 5 * 64, 1, (4, 4, 64)),
                                            (3 * 65 * 65, 192, 65 * 65, (64, 64, 192))])
def test_norm_backward_passes(rows, C, rpg, zp):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(rows, C, generator=g) * 0.7 + 0.3).to(BF16)
    du = torch.randn(rows, C, generator=g).to(BF16)
    if zp is not None:  # ZP pads are zero in both tensors
        H, W, Cch = zp
        e = torch.arange(rpg * C) // Cch
        pad = (((e // (W + 1)) == H) | ((e % (W + 1)) == W)).reshape(1, -1)
        x = torch.where(pad, torch.zeros((), dtype=BF16), x.reshape(-1, rpg * C)).reshape(rows, C)
        du = torch.where(pad, torch.zeros((), dtype=BF16), du.reshape(-1, rpg * C)).reshape(rows, C)
        count = H * W * Cch
    else:
        count = rpg * C
    G = rows // rpg
    xs = x.float().reshape(G, -1)
    mean = xs.sum(1) / count
    var = (xs * xs).sum(1) / count - mean * mean
    mr = torch.stack([mean, 1 / torch.sqrt(var + 1e-5)], 1)
    gamma = torch.randn(C, generator=g) * 0.3 + 1
    add = torch.randn(rows, C, generator=g).to(BF16)
    ms_e = E.group_sums(du, x, mr, gamma, rpg, count)
    ms = ops.group_sums(du.to(DEV), x.to(DEV), mr.to(DEV), gamma.to(DEV), rpg, count)
    assert torch.allclose(ms.cpu(), ms_e, rtol=2e-4, atol=2e-6)
    cs_e = E.col_sums(du, x, mr, rpg)
    cs = ops.col_sums(du.to(DEV), x.to(DEV), mr.to(DEV), rpg)
    assert rel(cs, cs_e) < 1e-5
    assert rel(ops.col_sums(du.to(DEV))[1], cs_e[1]) < 1e-5
    if rpg > 1:
        cs2, ms2 = ops.norm_sums(du.to(DEV), x.to(DEV), mr.to(DEV), gamma.to(DEV), rpg, count)
        assert rel(cs2, cs_e) < 1e-5 and torch.allclose(ms2.cpu(), ms_e, rtol=2e-4, atol=2e-6)
    dx_e = E.norm_bwd_apply(du, x, mr, gamma, ms_e, rpg, zp=zp, add=add)
    dx = ops.norm_bwd_apply(du.to(DEV), x.to(DEV), mr.to(DEV), gamma.to(DEV), ms_e.to(DEV), rpg, zp=zp, add=add.to(DEV))
    assert rel(dx, dx_e) < 4e-3 and (dx.float().cpu() - dx_e.float()).abs().max() <= 2 ** -7 * dx_e.float().abs().max()
    xr = x.float().relu().to(BF16)  # a ReLU output as the norm input: its backward is fused into the apply pass
    dxr_e = E.norm_bwd_apply(du, xr, mr, gamma, ms_e, rpg, zp=zp, relu_x=True)
    dxr = ops.norm_bwd_apply(du.to(DEV), xr.to(DEV), mr.to(DEV), gamma.to(DEV), ms_e.to(DEV), rpg, zp=zp, relu_x=True)
    assert rel(dxr, dxr_e) < 4e-3 and ((dxr.cpu() == 0) | (xr > 0)).all()
    if zp is not None:
        d4 = dx.cpu().reshape(G, zp[0] + 1, zp[1] + 1, -1)
        assert (d4[:, -1] == 0).all() and (d4[:, :, -1] == 0).all()


def test_maxpool_backward_with_ties():
    g = torch.Generator().manual_seed(3)
    # coarse values -> many exact ties inside windows; ~half the inputs are zero (post-ReLU)
    x = E.to_zp((torch.randint(-3, 4, (3, 16, 16, 64), generator=g).float().relu() * 0.5).to(BF16))
    dy = zp_rand(3, 8, 8, 64, g)
    ref = E.maxpool3s2_bwd(dy, x)
    out = ops.maxpool3s2_bwd(dy.to(DEV), x.to(DEV))
    assert torch.equal(out.cpu(), ref)


def test_firstconv_backward():
    g = torch.Generator().manual_seed(4)
    C0, F_, H, W = 64, 3, 32, 32
    img = torch.randint(0, 256, (F_, H, W, 3), dtype=torch.uint8, generator=g)
    w = (torch.randn(C0, 27, generator=g) * 0.2 / 255.0)
    b = torch.randn(C0, generator=g) * 0.1
    dy = zp_rand(F_, H // 2, W // 2, C0, g)
    dW_e, db_e = E.firstconv_bwd(img, w, b, dy, C0)
    dW, db = ops.firstconv_bwd(img.to(DEV), w.to(DEV), b.to(DEV), dy.to(DEV), C0)
    assert rel(dW, dW_e) < 2e-3 and rel(db, db_e) < 2e-3  # an arg-max of two nearly equal fp32 conv outputs may differ


@pytest.mark.parametrize("B,t,maxlen,heads,with_mem", [(2, 8, 8, 2, False), (3, 16, 8, 2, True), (2, 128, 128, 2, True)])
def test_attention_backward(B, t, maxlen, heads, with_mem):
    g = torch.Generator().manual_seed(5)
    h, T, nb = heads * 128, maxlen + t, 10
    q = (torch.randn(B * t, h, generator=g) * 3).to(BF16)
    kf = torch.randn(B, T, h, generator=g).to(BF16)
    vf = torch.randn(B, T, h, generator=g).to(BF16)
    R = torch.randn(B * t, heads * nb, generator=g)
    b_nd = torch.randn(nb, maxlen, generator=g) * 0.2
    first = torch.zeros(B, t, dtype=torch.uint8)
    smask = None
    if with_mem:
        smask = (torch.rand(B, 1, maxlen, generator=g) > 0.3).to(torch.uint8)
        first[0, 0] = 1  # batch row 0 forgets its memory
    dO = torch.randn(B * t, h, generator=g).to(BF16)
    ld = (3 * h + heads * nb + 7) // 8 * 8
    out_e = torch.zeros(B * t, ld, dtype=BF16)
    db_e = E.attention_bwd(q, kf, vf, R, b_nd, first, smask, dO, out_e, B, t, maxlen, heads)
    out = torch.zeros(B * t, ld, dtype=BF16, device=DEV)
    db = ops.attention_bwd(q.to(DEV), kf.to(DEV), vf.to(DEV), R.to(DEV), b_nd.to(DEV), first.to(DEV), None if smask is None else smask.to(DEV),
                           dO.to(DEV), out, B, t, maxlen, heads)
    nat.device_check()
    for name, sl in [("dq", slice(0, h)), ("dk", slice(h, 2 * h)), ("dv", slice(2 * h, 3 * h)), ("dR", slice(3 * h, 3 * h + heads * nb))]:
        assert rel(out[:, sl], out_e[:, sl]) < 6e-3, name
    assert rel(db, db_e) < 1e-3


def test_softmax_backward():
    g = torch.Generator().manual_seed(6)
    logp = torch.log_softmax(torch.randn(37, 121, generator=g), -1)
    idx = torch.randint(0, 121, (37,), generator=g)
    out_e = torch.zeros(37, 136, dtype=BF16)
    E.softmax_bwd(logp, idx, 0.25, out_e, 8)
    out = torch.zeros(37, 136, dtype=BF16, device=DEV)
    ops.softmax_bwd(logp.to(DEV), idx.to(DEV), 0.25, out, 8)
    assert rel(out, out_e) < 4e-3 and (out[:, :8] == 0).all() and (out[:, 129:] == 0).all()


def _case(seed=0, B=2, T=8):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    return img, first, actions


def test_bc_step_matches_emulated_step_and_oracle_direction():
    """Same weights, same batch: (a) the CUDA step against the emulated step (same bf16 rounding points, so the ReLU / pool masks
    agree except where accumulation order moves a value across zero), (b) against autograd through the fp32 oracle, where only
    the direction is comparable (see tests/test_training.py)."""
    pol, sd, cfg = make_policy(small_kwargs())
    img, first, actions = _case()
    with emulation():
        tr_e = BCTrainer(pol)
        loss_e, _ = tr_e.loss_and_grad(img, first, pol.initial_state(2), actions)
    grads_e = {n: p.grad.clone() for n, p in pol.named_parameters() if p.grad is not None}
    for p in pol.parameters():
        p.grad = None
    pol = pol.to(DEV)
    tr = BCTrainer(pol)
    loss, st = tr.loss_and_grad(img.to(DEV), first.to(DEV), pol.initial_state(2), {k: v.to(DEV) for k, v in actions.items()})
    nat.device_check()
    assert abs(loss.item() - loss_e.item()) < 2e-3 * abs(loss_e.item())
    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    (pd, _, _), _ = O.agent_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    loss_o = -O.logprob(pd, actions).mean()
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-2 * abs(loss_o.item())
    errs, coss = {}, {}
    for n, p in pol.named_parameters():
        if n.startswith("value_head"):
            assert p.grad is None
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        errs[n] = rel(p.grad, grads_e[n])
        g_o = leaf[n].grad
        coss[n] = ((p.grad.cpu() * g_o).sum() / (p.grad.cpu().norm() * g_o.norm())).item()
    print("rel-L2 vs emulated step:", " ".join(f"{e:.3f}" for e in errs.values()))
    print("cosine vs oracle autograd:", " ".join(f"{c:.3f}" for c in coss.values()))
    # Two bf16 forwards with different summation orders decorrelate by ~1 % after a few layers, and every ReLU / max-pool mask
    # between the loss and a parameter turns that into ~10 % gradient noise (tests/test_training.py), so only the parameters
    # right below the loss can be compared tightly; for the rest the measure is the direction against the exact gradient
    # (measured: cosine 0.93-0.96 in stack 0, > 0.98 in the transformer, 1.000 at the heads).
    for n, e in errs.items():
        top = n.startswith("pi_head") or n.startswith("net.final_ln")
        assert e < (0.05 if top else 0.6), (n, e)
    for n, c in coss.items():
        assert c > 0.85, (n, c)


def test_cuda_backward_matches_autograd_at_the_taped_operating_point():
    """The tight pin of the CUDA backward (VERDICT round 1, weak 1; ADVICE): the CUDA forward's taped activations are fed into the
    forced torch-autograd replica (tests/forced_replica.py: fp32 layers from the parameters, values and ReLU / max-pool masks
    forced from the tape, on the same GPU with TF32 off), so the comparison isolates the backward kernels -- dgrad / wgrad with bf16
    operands, norm / pool / attention / softmax backward -- from forward mask flips.  Per-parameter rel-L2 < 3e-2."""
    from forced_replica import forced_loss

    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        for kw, B, T, seed in [(small_kwargs(), 2, 8, 0), (small_kwargs(timesteps=24, attention_memory_size=40), 3, 24, 3)]:
            pol, sd, cfg = make_policy(kw, seed=seed)
            g = torch.Generator().manual_seed(seed)
            img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g).to(DEV)
            first = torch.zeros(B, T, dtype=torch.bool, device=DEV)
            actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).to(DEV), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).to(DEV)}
            pol = pol.to(DEV)
            tr = BCTrainer(pol)
            tr.keep_tape = True
            state = pol.initial_state(B)
            if seed:  # second case: a filled KV memory (detached constants in the backward) and a mid-batch episode start
                (_, _, _), state = pol({"img": img}, first, state)
                first = first.clone()
                first[1, 0] = True
            loss, _ = tr.loss_and_grad(img, first, state, actions)
            nat.device_check()
            leaf = {k: v.to(DEV).clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
            lf = forced_loss(leaf, cfg, tr.last_tape, img, first, actions)
            lf.backward()
            assert abs(loss.item() - lf.item()) < 1e-3 * abs(lf.item()), (loss.item(), lf.item())
            errs = {}
            for n, p in pol.named_parameters():
                if n.startswith("value_head"):
                    assert p.grad is None
                    continue
                errs[n] = rel(p.grad, leaf[n].grad)
            top = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
            print(f"B={B} T={T}: worst rel-L2 vs forced autograd: " + ", ".join(f"{n} {e:.4f}" for n, e in top))
            # measured: <= 1.3e-2 for every parameter except the stack-0 / stack-1 post-pool norms (2.3e-2: their dgamma sums ~10^5
            # bf16-rounded products per channel); the CPU emulation of the same rounding points gives 1.6e-2 at worst (test_training.py)
            for n, e in errs.items():
                assert e < 3e-2, (n, e)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_bc_training_reduces_the_loss():
    """A few full steps (forward, backward, flat-bucket Adam) on one fixed batch must drive the NLL down."""
    pol, _, _ = make_policy(small_kwargs())
    pol = pol.to(DEV)
    img, first, actions = _case(seed=1, B=4)
    img, first = img.to(DEV), first.to(DEV)
    actions = {k: v.to(DEV) for k, v in actions.items()}
    tr = BCTrainer(pol)
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=2e-4)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(4), actions)
        opt.step()
        losses.append(loss.item())
    nat.device_check()
    assert all(l == l for l in losses) and losses[-1] < losses[0] - 0.5, losses


def test_graphed_policy_relayout_equals_eager():
    """The policy's refresh_weights: from the second optimizer step on the kernel-side weight re-layout is one CUDA-graph replay; the
    training trajectory must be bit-identical to the eager re-layout."""
    img, first, actions = _case(seed=2, B=2)
    img, first = img.to(DEV), first.to(DEV)
    actions = {k: v.to(DEV) for k, v in actions.items()}
    finals = []
    for graphed in (False, True):
        pol, _, _ = make_policy(small_kwargs(), seed=4)
        pol = pol.to(DEV)
        tr = BCTrainer(pol)
        pol.graph_relayout = graphed
        opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=2e-4)
        losses = []
        for _ in range(5):
            opt.zero_grad()
            loss, _ = tr.loss_and_grad(img, first, pol.initial_state(2), actions)
            opt.step()
            losses.append(loss.item())
        assert (pol._relayout is not None) == graphed
        finals.append((losses, opt.flat_p.clone()))
    nat.device_check()
    assert finals[0][0] == finals[1][0], (finals[0][0], finals[1][0])
    assert torch.equal(finals[0][1], finals[1][1])


def test_bc_and_rl_steps_share_one_relayout_graph():
    """BC and RL steps alternating on one policy with FlatAdamDP: the policy holds one re-layout graph, which rewrites both trainers'
    heads_t as well, and the trajectory (losses, parameters, EWMA normaliser) is bit-identical to the eager re-layout."""
    B, T = 2, 8
    img, first, actions = _case(seed=3, B=B, T=T)
    img, first = img.to(DEV), first.to(DEV)
    actions = {k: v.to(DEV) for k, v in actions.items()}
    g = torch.Generator().manual_seed(5)
    old = (0.1 * torch.randn(B, T, generator=g) - 14.0).to(DEV)  # ~ log(1/121) + log(1/8641): ratios near 1
    adv, returns = torch.randn(B, T, generator=g).to(DEV), (3.0 + torch.randn(B, T, generator=g)).to(DEV)
    finals = []
    for graphed in (False, True):
        pol, _, _ = make_policy(small_kwargs(), seed=4)
        pol = pol.to(DEV)
        pol.graph_relayout = graphed
        bc, rl = BCTrainer(pol), RLTrainer(pol)
        opt = FlatAdamDP(pol.parameters(), lr=2e-4)  # (the normaliser does not require grad: not in the bucket)
        losses = []
        for i in range(6):
            opt.zero_grad()
            if i % 2 == 0:
                loss, _ = bc.loss_and_grad(img, first, pol.initial_state(B), actions)
            else:
                loss, _ = rl.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, vf_coef=0.5, kl_coef=0.0)
            opt.step()
            losses.append(loss.item())
        # one graph: the net's forward folds and backward transposes, the head folds, BC's and RL's heads_t
        assert (pol._relayout is not None and len(pol._relayout[1]) == 5) if graphed else pol._relayout is None
        finals.append((losses, opt.flat_p.clone(), pol.value_head.normalizer.running_mean.clone()))
    nat.device_check()
    assert finals[0][0] == finals[1][0], (finals[0][0], finals[1][0])
    assert torch.equal(finals[0][1], finals[1][1]) and torch.equal(finals[0][2], finals[1][2])


def test_bc_step_at_3x_width_shapes():
    """BASELINE configs[3] layer shapes (3x: 192/384/384 channels, hidsize 3072, 24 heads, 128-frame memory, 128x128 frames) on
    a short clip: every backward kernel runs at its production shape, gradients are finite and Adam steps lower the loss."""
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("3x"), vpt_b200.PI_HEAD_KWARGS).to(DEV)
    g = torch.Generator().manual_seed(7)
    B, T = 2, 8
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).to(DEV)
    first = torch.zeros(B, T, dtype=torch.bool, device=DEV)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).to(DEV), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).to(DEV)}
    tr = BCTrainer(pol)
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=1e-4)
    state, losses = pol.initial_state(B), []
    for _ in range(4):
        opt.zero_grad()
        loss, state = tr.loss_and_grad(img, first, state, actions)  # the KV memory is carried (and detached) across steps
        assert torch.isfinite(opt.flat_g).all()
        opt.step()
        losses.append(loss.item())
    nat.device_check()
    assert losses[-1] < losses[0], losses
