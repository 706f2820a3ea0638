"""`recompute_frames` on the H100 at the released models' shapes: the backward re-runs the ImpalaCNN chunk by chunk instead of keeping its
activations.  Against the stored-tape path on the same batch (bit for bit with one chunk), one large call against the sum of the stored-tape
calls it replaces, and a 3x BPTT window that the stored tape cannot hold.  tests/test_recompute.py checks the same on the CPU emulation
against the oracle's exact gradient."""
import pytest
import torch

import vpt_b200
from common import perturb
from video_pre_training_b200 import _native as nat
from video_pre_training_b200.parallel import FlatAdamDP
from video_pre_training_b200.training import BCTrainer, IDMTrainer

pytestmark = pytest.mark.gpu


def _policy(width):
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    return pol.cuda()


def _frames(g, B, T=128):
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    return img, torch.zeros(B, T, dtype=torch.bool).cuda(), actions


def _take(grads, mod):
    """Moves the parameters' .grad into `grads` (summed), leaving .grad None."""
    for n, p in mod.named_parameters():
        if p.grad is not None:
            grads[n] = p.grad if n not in grads else grads[n].add_(p.grad)
            p.grad = None
    return grads


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300)).item()


def _step(pol, tr, img, first, actions):
    loss, st = tr.loss_and_grad(img, first, pol.initial_state(img.shape[0]), actions)
    nat.device_check()
    return loss, st, _take({}, pol)


def test_2x_bc_one_chunk_is_bit_identical():
    """2x BC at B = 16, T = 128 (2048 frames): recompute_frames = 2048 re-runs the forward's one CNN chunk with the same launches, so the loss,
    every gradient and state_out are those of the stored tape bit for bit."""
    pol = _policy("2x")
    img, first, actions = _frames(torch.Generator().manual_seed(0), 16)
    l0, s0, g0 = _step(pol, BCTrainer(pol), img, first, actions)
    l1, s1, g1 = _step(pol, BCTrainer(pol, recompute_frames=2048), img, first, actions)
    assert torch.equal(l0, l1)
    assert g0.keys() == g1.keys() and not any(n.startswith("value_head") for n in g0)
    for n in g0:
        assert torch.equal(g0[n], g1[n]), (n, _rel(g1[n], g0[n]))
    for (_, (k0, v0)), (_, (k1, v1)) in zip(s0, s1):
        assert torch.equal(k0, k1) and torch.equal(v0, v1)


def test_2x_bc_512_frame_chunks():
    """The same batch in CNN chunks of 512 frames.  512 is a multiple of the conv's 128-row M tile and a frame of every stack is a whole
    number of rows, so every tile starts at the same pixel of the same frame as in the 2048-frame launch, and the recomputed CNN output and
    its statistics equal the stored ones bit for bit: everything above the CNN is bit-identical.  Inside the CNN the backward's reductions
    over frames (weight gradients, per-channel sums) are split over four launches whose partial sums add in fp32, and the norm backward's
    per-frame sums are split into slabs by frame count, so those parameters differ by fp32 reassociation and the bf16 roundings it moves."""
    pol = _policy("2x")
    img, first, actions = _frames(torch.Generator().manual_seed(0), 16)
    tr0 = BCTrainer(pol)
    tr0.keep_tape = True
    l0, _, g0 = _step(pol, tr0, img, first, actions)
    out0 = tr0.last_tape["cnn_out"]
    tr0.last_tape = None
    tr1 = BCTrainer(pol, recompute_frames=512)
    seen = []
    tr1.on_recompute = lambda f0, f1, out, mr: seen.append(torch.equal(out, out0[f0:f1]))
    l1, _, g1 = _step(pol, tr1, img, first, actions)
    assert seen == [True] * 4
    assert torch.equal(l0, l1)
    worst = {}
    for n in g0:
        if n.startswith("net.img_process.cnn.stacks."):
            worst[n] = _rel(g1[n], g0[n])
        else:
            assert torch.equal(g0[n], g1[n]), (n, _rel(g1[n], g0[n]))
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("2x B=16 in 512-frame CNN chunks vs the stored tape, CNN parameters, worst rel-L2", top)
    assert top[0][1] < 1e-2  # measured 2.63e-3 (H100); fp32 reassociation alone would be ~1e-6, the moved bf16 roundings of dx dominate


def test_2x_bc_b128_in_one_call():
    """2x BC at B = 128, T = 128 (16384 frames) in one call against eight stored-tape calls of B = 16 on the same sequences.  The loss of the
    big call is the mean of the eight and its logits gradient exactly 1/8 of theirs (a power of two: the same bf16 roundings), the CNN runs
    in the same 2048-frame chunks; what differs is where the sums over frames are split (the weight-gradient GEMMs and column sums over 16384
    rows against eight fp32 `.grad` additions), i.e. fp32 reassociation."""
    pol = _policy("2x")
    g = torch.Generator().manual_seed(1)
    parts = [_frames(g, 16) for _ in range(8)]
    tr = BCTrainer(pol)
    ref, losses = {}, []
    for img, first, actions in parts:
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(16), actions)
        losses.append(loss.item())
        _take(ref, pol)
    del tr
    img = torch.cat([p[0] for p in parts])
    first = torch.cat([p[1] for p in parts])
    actions = {k: torch.cat([p[2][k] for p in parts]) for k in parts[0][2]}
    del parts
    torch.cuda.reset_peak_memory_stats()
    loss, _ = BCTrainer(pol, recompute_frames=2048).loss_and_grad(img, first, pol.initial_state(128), actions)
    nat.device_check()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    big = _take({}, pol)
    assert abs(loss.item() - sum(losses) / 8) < 1e-5 * abs(loss.item())
    assert big.keys() == ref.keys()
    worst = {n: _rel(8 * big[n], ref[n]) for n in ref if ref[n].any()}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"2x B=128 T=128 one call (peak {peak:.1f} GiB) vs 8 x B=16 stored-tape calls, worst rel-L2", top)
    assert top[0][1] < 1e-3  # measured 5.96e-5 (pi_head.buttons weight; H100), peak 57.5 GiB


def test_4x_idm_b16_in_one_call():
    """The released 4x IDM at B = 16, T = 128 (2048 frames) in one call, CNN chunks of four sequences, against four stored-tape calls of
    B = 4; as above, the differences are where the frame sums are split (the loss scale differs by exactly 4)."""
    torch.manual_seed(0)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs())
    perturb(pol)
    pol = pol.cuda()
    g = torch.Generator().manual_seed(2)
    img = torch.randint(0, 256, (16, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(16, 128, dtype=torch.bool).cuda()
    actions = {"buttons": torch.randint(0, 2, (16, 128, 20), generator=g).cuda(), "camera": torch.randint(0, 11, (16, 128, 2), generator=g).cuda()}
    tr = IDMTrainer(pol)
    ref, losses = {}, []
    for b in range(0, 16, 4):
        loss, _ = tr.loss_and_grad(img[b:b + 4], first[b:b + 4], pol.initial_state(4), {k: v[b:b + 4] for k, v in actions.items()})
        losses.append(loss.item())
        _take(ref, pol)
    tr = IDMTrainer(pol, recompute_frames=512)
    chunks = []
    tr.on_recompute = lambda f0, f1, out, mr: chunks.append((f0, f1))
    loss, _ = tr.loss_and_grad(img, first, pol.initial_state(16), actions)
    nat.device_check()
    big = _take({}, pol)
    assert chunks == [(1536, 2048), (1024, 1536), (512, 1024), (0, 512)]
    assert abs(loss.item() - sum(losses) / 4) < 1e-5 * abs(loss.item())
    assert big.keys() == ref.keys()
    worst = {n: _rel(4 * big[n], ref[n]) for n in ref if ref[n].any()}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("4x IDM B=16 T=128 one call vs 4 x B=4 stored-tape calls, worst rel-L2", top)
    assert top[0][1] < 1e-3  # measured 2.61e-6 (H100)


def test_3x_bptt_window_of_four_chunks():
    """A 3x truncated-BPTT window of four B = 16, T = 128 calls (8192 frames in one graph) with CNN chunks of 512 frames: one backward
    and one FlatAdamDP step.  The stored tape holds about 25 MB per frame at 3x and does not fit one such window."""
    pol = _policy("3x").set_autograd(True, state_grad=True, recompute_frames=512)
    g = torch.Generator().manual_seed(3)
    chunks = [_frames(g, 16) for _ in range(4)]
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=1e-5)
    torch.cuda.reset_peak_memory_stats()
    st, loss = pol.initial_state(16), 0.0
    for img, first, actions in chunks:
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss - pol.logprob(actions, pd).mean()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    nat.device_check()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"3x BPTT window of 4 x (B=16, T=128), recompute_frames=512: loss {loss.item():.4f}, peak {peak:.1f} GiB")
    assert torch.isfinite(loss)
    assert all(torch.isfinite(p).all() for p in pol.parameters())
    assert dict(pol.named_parameters())["net.img_process.cnn.stacks.0.firstconv.layer.weight"].grad.abs().sum() > 0
