"""Truncated BPTT across calls on the H100: `vpt_attention_bwd_state` against the float64 closed form of tests/bptt_refs.py (itself checked
against torch autograd on the CPU by tests/test_bptt.py), and `loss.backward()` over windows of chunks with the state attached against the
emulated CPU step and against the BPTT forced replica (tests/forced_replica_bptt.py) at the SMALL config and at 2x width."""
import contextlib

import pytest
import torch

import bptt_refs
import emu_autograd_ops
import emu_bptt_ops
import emu_idm_ops
import emu_ops
import vpt_b200
from common import make_policy, perturb, small_kwargs
from test_autograd import batch, bc_loss
from test_bptt import window_vs_forced
from test_gpu_rl_training import no_tf32
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP

pytestmark = pytest.mark.gpu

GUARD = 0xFFFF  # bf16 NaN pattern of the guard columns
PAD = 64        # fp32 NaN guard elements before and after each dmem buffer


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300)).item()


def _call(x, B, t, maxlen, heads, dstate, want_dmem, ld):
    """One vpt_attention_bwd_state launch through the C ABI with NaN guard columns right of `out` and NaN guard bands around dmem."""
    h = heads * 128
    out = torch.full((B * t, ld), -1, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    db = torch.empty(10, maxlen, dtype=torch.float32, device="cuda")
    ws = torch.empty(2 * B * heads * t * maxlen, dtype=torch.float32, device="cuda")
    n = B * maxlen * h
    bufs = [torch.full((n + 2 * PAD,), float("nan"), device="cuda") for _ in range(2)] if want_dmem else None
    ptr = lambda a: None if a is None else a.data_ptr()  # noqa: E731
    R = x["R"]
    nat.check(nat.lib().vpt_attention_bwd_state(ptr(x["Q"]), ptr(x["Kf"]), ptr(x["Vf"]), ptr(R), R.stride(0), ptr(x["b_nd"]), ptr(x["first_u8"]),
                                                x["first_u8"].stride(0), ptr(x["smask_u8"]), ptr(x["dO"]), ptr(out), ld, ptr(db), ptr(ws), B, t,
                                                maxlen, heads, 10, ptr(dstate[0]), ptr(dstate[1]),
                                                None if bufs is None else bufs[0].data_ptr() + 4 * PAD,
                                                None if bufs is None else bufs[1].data_ptr() + 4 * PAD, None), "vpt_attention_bwd_state")
    torch.cuda.synchronize()
    return out, db, bufs


@pytest.mark.parametrize("B,t,maxlen,heads", [(16, 128, 128, 16), (2, 128, 128, 24), (64, 1, 128, 16), (4, 37, 128, 8)])
@pytest.mark.parametrize("with_dstate", [True, False])
def test_kernel_matches_float64(B, t, maxlen, heads, with_dstate):
    x = bptt_refs.inputs(B, t, maxlen, heads, seed=B + t + heads, dev="cuda", with_dstate=with_dstate)
    h = heads * 128
    nr = 10 * heads
    ld = (3 * h + nr + 7) // 8 * 8 + 16
    cpu = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in x.items()}
    ref = bptt_refs.closed_form(cpu["Q"], cpu["Kf"], cpu["Vf"], cpu["R"], cpu["b_nd"], cpu["first_u8"], cpu["smask_u8"], cpu["dO"], B, t, maxlen,
                                heads, dstate=tuple(None if d is None else d.cpu() for d in x["dstate"]))
    runs = [_call(x, B, t, maxlen, heads, x["dstate"], True, ld) for _ in range(2)]
    out, db, bufs = runs[0]
    o = out.cpu()
    raw = o.view(torch.int16).to(torch.int32) & 0xFFFF
    assert (raw[:, 3 * h + nr:] == GUARD).all(), "guard columns written"
    for buf in bufs:
        assert torch.isnan(buf[:PAD]).all() and torch.isnan(buf[-PAD:]).all(), "dmem guard band written"
        assert torch.isfinite(buf[PAD:-PAD]).all(), "dmem not written in full"
    got = dict(dq=o[:, :h], dk=o[:, h:2 * h], dv=o[:, 2 * h:3 * h], dR=o[:, 3 * h:3 * h + nr], db_nd=db.cpu(),
               dmem_k=bufs[0][PAD:-PAD].cpu().view(B, maxlen, h), dmem_v=bufs[1][PAD:-PAD].cpu().view(B, maxlen, h))
    errs = {k: _rel(got[k], ref[k]) for k in got}
    print(f"B={B} t={t} heads={heads} dstate={with_dstate}:", {k: f"{e:.2e}" for k, e in errs.items()})
    # bf16 outputs: one bf16 rounding; the fp32 ones: fp32 accumulation.  Worst measured over the eight cases (H100): bf16 1.70e-3,
    # fp32 3.69e-7 (d b_nd; dmem 3.58e-7)
    for k in ("dq", "dk", "dv", "dR"):
        assert errs[k] < 6.8e-3, (k, errs[k])
    for k in ("db_nd", "dmem_k", "dmem_v"):
        assert errs[k] < 1.4e-6, (k, errs[k])
    # bit-reproducible
    o2, db2, bufs2 = runs[1]
    assert torch.equal(out.view(torch.int16), o2.view(torch.int16)) and torch.equal(db, db2)
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(bufs, bufs2))
    # without a state gradient: every column bit-identical to vpt_attention_bwd, with or without dmem
    args = (x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], x["dO"])
    base = torch.zeros(B * t, ld, dtype=torch.bfloat16, device="cuda")
    db0 = ops.attention_bwd(*args, base, B, t, maxlen, heads)
    for want in (False, True):
        o3 = torch.zeros_like(base)
        db3, dm = ops.attention_bwd_state(*args, o3, B, t, maxlen, heads, dstate=None, want_dmem=want)
        assert torch.equal(o3.view(torch.int16), base.view(torch.int16)) and torch.equal(db3, db0)
        assert (dm is None) == (not want)
    if not with_dstate:
        assert torch.equal(out[:, :3 * h + nr].view(torch.int16), base[:, :3 * h + nr].view(torch.int16))
    # the wrapper gives the C call's bits
    o4 = torch.zeros_like(base)
    _, (dk4, dv4) = ops.attention_bwd_state(*args, o4, B, t, maxlen, heads, dstate=x["dstate"], want_dmem=True)
    assert torch.equal(o4[:, :3 * h + nr].view(torch.int16), out[:, :3 * h + nr].view(torch.int16))
    assert torch.equal(dk4.view(-1), bufs[0][PAD:-PAD]) and torch.equal(dv4.view(-1), bufs[1][PAD:-PAD])


def test_wrapper_refuses_bad_state_gradients():
    x = bptt_refs.inputs(2, 8, 16, 1, seed=0, dev="cuda")
    args = (x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], x["dO"])
    out = torch.zeros(16, 3 * 128 + 16, dtype=torch.bfloat16, device="cuda")
    dk = x["dstate"][0]
    for bad in ((dk.double(), None), (dk[:, :8].contiguous(), None), (None, dk.transpose(1, 2).contiguous().transpose(1, 2)), (dk,)):
        with pytest.raises(ValueError):
            ops.attention_bwd_state(*args, out, 2, 8, 16, 1, dstate=bad)


@contextlib.contextmanager
def _emulated():
    """ops routed through the CPU emulation for the duration (the same routing as the `bptt` fixture of tests/test_bptt.py)."""
    saved = {}
    for mod in (emu_ops, emu_idm_ops, emu_autograd_ops, emu_bptt_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                fn = getattr(mod, name)
                if name in ("maxpool3s2_bwd", "firstconv_bwd", "attention_bwd", "conv3d_t5_bwd", "attention_bwd_state"):
                    fn = (lambda f: lambda *a, **k: _grad_on(f, *a, **k))(fn)
                saved.setdefault(name, getattr(ops, name))
                setattr(ops, name, fn)
    try:
        yield
    finally:
        for name, fn in saved.items():
            setattr(ops, name, fn)


def _grad_on(fn, *a, **k):
    with torch.enable_grad():
        return fn(*a, **k)


def _window_grads(pol, chunks, dev):
    st = pol.initial_state(chunks[0][0].shape[0])
    loss = 0.0
    for img, first, actions in chunks:
        (pd, _, _), st = pol({"img": img.to(dev)}, first.to(dev), st)
        loss = loss + bc_loss(pol, pd, {k: v.to(dev) for k, v in actions.items()})
    loss.backward()
    return loss.item(), {n: None if p.grad is None else p.grad.cpu() for n, p in pol.named_parameters()}


def test_small_two_chunks_vs_emulation_and_forced_replica():
    g = torch.Generator().manual_seed(7)
    chunks = [batch(g, 2, 8, reset=(1, 0) if c == 1 else None) for c in range(2)]
    pol_c, _, _ = make_policy(small_kwargs())
    with _emulated():
        loss_c, grads_c = _window_grads(pol_c.set_autograd(True, state_grad=True), chunks, "cpu")
    pol, sd, cfg = make_policy(small_kwargs())
    pol = pol.cuda().set_autograd(True, state_grad=True)
    loss, grads = _window_grads(pol, chunks, "cuda")
    nat.device_check()
    worst = {}
    for n, gc in grads_c.items():
        assert (grads[n] is None) == (gc is None), n
        if gc is not None and gc.any():
            worst[n] = _rel(grads[n], gc)
    rest = sorted(((n, e) for n, e in worst.items() if ".cnn." not in n), key=lambda kv: -kv[1])[:4]
    print("small two chunks: CUDA vs emulated CPU step, worst", rest, "outside the CNN; loss", loss, loss_c)
    assert abs(loss - loss_c) < 1e-2 * abs(loss_c)
    # The two bf16 forwards round differently, so ReLU / max-pool masks flip and the peaked attention of the perturbed weights (q x 30)
    # moves: measured (H100) up to 0.30 rel-L2 in the CNN and 0.26 outside it (b_nd, r_layer).  Against the emulation the loss and the None
    # pattern are pinned; the gradients are pinned by the forced replica below, at the CUDA forward's operating point.
    pol.zero_grad(set_to_none=True)
    cuda_chunks = [(img.cuda(), first.cuda(), {k: v.cuda() for k, v in a.items()}) for img, first, a in chunks]
    loss, loss_f, worst = window_vs_forced(pol, {k: v.cuda() for k, v in sd.items()}, cfg, cuda_chunks, (0, 1), ctx=no_tf32)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("small two chunks: CUDA vs BPTT forced replica, worst", top)
    assert abs(loss - loss_f) < 1e-3 * abs(loss_f)
    assert top[0][1] < 3e-2  # measured 1.38e-2 (H100)


def _policy_2x():
    kw = vpt_b200.policy_kwargs("2x", n_recurrence_layers=4)
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    sd = {k: v.detach().clone().cuda() for k, v in pol.state_dict().items()}
    import vpt_oracle as O
    return pol.cuda(), sd, O.Cfg(**kw)


def _frames(g, B, T):
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    return img, torch.zeros(B, T, dtype=torch.bool).cuda(), actions


def test_2x_two_full_chunks_vs_forced_replica():
    pol, sd, cfg = _policy_2x()
    pol.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(8)
    chunks = [_frames(g, 2, 128) for _ in range(2)]
    chunks[1][1][1, 0] = True
    loss, loss_f, worst = window_vs_forced(pol, sd, cfg, chunks, (0, 1), ctx=no_tf32)
    nat.device_check()
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("2x B=2 T=128 x 2 chunks vs BPTT forced replica, worst", top)
    assert abs(loss - loss_f) < 1e-3 * abs(loss_f)
    assert top[0][1] < 3e-2  # measured 1.32e-2 (H100)


def test_2x_one_frame_loop_vs_forced_replica():
    """The reference loop's shape (B = 1, T = 1) over four calls, one backward, after a 128-frame inference chunk filled the memory."""
    pol, sd, cfg = _policy_2x()
    g = torch.Generator().manual_seed(9)
    img0 = torch.randint(0, 256, (1, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    with torch.no_grad():
        _, st = pol({"img": img0}, torch.zeros(1, 128, dtype=torch.bool).cuda(), pol.initial_state(1))
    pol.set_autograd(True, state_grad=True)
    chunks = [_frames(g, 1, 1) for _ in range(4)]
    loss, loss_f, worst = window_vs_forced(pol, sd, cfg, chunks, (0, 1, 2, 3), ctx=no_tf32, st=st)
    nat.device_check()
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("2x B=1 T=1 x 4 calls vs BPTT forced replica, worst", top)
    assert abs(loss - loss_f) < 1e-3 * abs(loss_f)
    assert top[0][1] < 3e-2  # measured 1.62e-2 (H100)


def test_adam_steps_on_a_two_chunk_window_lower_the_loss():
    pol, _, _ = make_policy(small_kwargs())
    pol = pol.cuda().set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(10)
    chunks = [tuple(x.cuda() if isinstance(x, torch.Tensor) else {k: v.cuda() for k, v in x.items()} for x in batch(g, 2, 8)) for _ in range(2)]
    params = [p for n, p in pol.named_parameters() if p.requires_grad and not n.startswith("value_head")]
    opt = FlatAdamDP(params, lr=3e-4)
    losses = []
    for _ in range(4):
        opt.zero_grad()
        st, loss = pol.initial_state(2), 0.0
        for img, first, actions in chunks:
            (pd, _, _), st = pol({"img": img}, first, st)
            loss = loss + bc_loss(pol, pd, actions)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print("two-chunk window losses", losses)
    assert losses[-1] < losses[0]
