"""Training part of a policy on the H100 at the released models' shapes: with the CNN frozen (or all but the heads) the trainable gradients,
the loss and state_out are those of the all-trainable step bit for bit, frozen `.grad` stays None, fewer kernels launch, the CNN tape is
not kept and a call is no longer bounded by it.  tests/test_freeze.py checks the same rules on the CPU emulation against the oracle."""
import pytest
import torch

import vpt_b200
from common import perturb
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.training import BCTrainer, IDMTrainer

pytestmark = pytest.mark.gpu

MiB = 2 ** 20


def _policy(width):
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    return pol.cuda()


def _frames(g, B, T=128):
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    return img, torch.zeros(B, T, dtype=torch.bool).cuda(), actions


def _freeze(mod, prefixes, keep=False):
    """requires_grad on the parameters whose names start with `prefixes` (keep=True: on all the others) off."""
    for n, p in mod.named_parameters():
        if n.startswith(prefixes) != keep:
            p.requires_grad_(False)


def _unfreeze(mod):
    for n, p in mod.named_parameters():
        p.requires_grad_(not n.startswith("value_head.normalizer."))


def _run(mod, tr, img, first, actions):
    """One call -> (loss, state_out, {name: .grad} (moved out), launches, peak bytes)."""
    for p in mod.parameters():
        p.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    n0 = ops.LAUNCHES
    loss, st = tr.loss_and_grad(img, first, mod.initial_state(img.shape[0]), actions)
    torch.cuda.synchronize()
    nat.device_check()
    launches, peak = ops.LAUNCHES - n0, torch.cuda.max_memory_allocated()
    grads = {}
    for n, p in mod.named_parameters():
        grads[n], p.grad = p.grad, None
    return loss, st, grads, launches, peak


def _same(a, b, frozen):
    """a: the partial run, b: the all-trainable one."""
    (l0, s0, g0, *_), (l1, s1, g1, *_) = a, b
    assert torch.equal(l0, l1)
    for (_, (k0, v0)), (_, (k1, v1)) in zip(s0, s1):
        assert torch.equal(k0, k1) and torch.equal(v0, v1)
    for n in g0:
        if n.startswith(frozen) or g1[n] is None:
            assert g0[n] is None, n
        else:
            assert g0[n] is not None and torch.equal(g0[n], g1[n]), n


def test_2x_bc_frozen_cnn_is_bit_identical_and_cheaper():
    """2x BC at B = 16, T = 128: the CNN (`img_process.cnn.*`) frozen against all trainable."""
    pol = _policy("2x")
    img, first, actions = _frames(torch.Generator().manual_seed(0), 16)
    full = _run(pol, BCTrainer(pol), img, first, actions)
    _freeze(pol, ("net.img_process.cnn.",))
    part = _run(pol, BCTrainer(pol), img, first, actions)
    _same(part, full, "net.img_process.cnn.")
    print(f"2x BC B=16 T=128: launches {full[3]} -> {part[3]}, peak {full[4] / 2 ** 30:.2f} -> {part[4] / 2 ** 30:.2f} GiB")
    assert part[3] < full[3]
    assert part[4] < full[4] - 2048 * 15 * MiB  # at least the CNN tape (20.7 MiB per frame with its backward workspace, README)


def test_2x_bc_frozen_cnn_4096_frames_in_one_call():
    """2x BC at B = 32, T = 128 (4096 frames) with the CNN frozen runs without recompute_frames, in the same 2048-frame CNN chunks as the
    all-trainable call with recompute_frames = 2048: the trainable gradients are bit-identical to that call's."""
    pol = _policy("2x")
    img, first, actions = _frames(torch.Generator().manual_seed(1), 32)
    full = _run(pol, BCTrainer(pol, recompute_frames=2048), img, first, actions)
    _freeze(pol, ("net.img_process.cnn.",))
    part = _run(pol, BCTrainer(pol), img, first, actions)
    _same(part, full, "net.img_process.cnn.")


def test_4x_idm_frozen_cnn_is_bit_identical_and_cheaper():
    """4x IDM at B = 4, T = 128 with the conv3d pre-stage and the CNN frozen against all trainable."""
    torch.manual_seed(0)
    idm = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()
    g = torch.Generator().manual_seed(2)
    img = torch.randint(0, 256, (4, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(4, 128, dtype=torch.bool).cuda()
    actions = {"buttons": torch.randint(0, 2, (4, 128, 20), generator=g).cuda(), "camera": torch.randint(0, 11, (4, 128, 2), generator=g).cuda()}
    full = _run(idm, IDMTrainer(idm), img, first, actions)
    frozen = ("net.img_process.cnn.", "net.conv3d_layer.")
    _freeze(idm, frozen)
    part = _run(idm, IDMTrainer(idm), img, first, actions)
    _same(part, full, frozen)
    print(f"4x IDM B=4 T=128: launches {full[3]} -> {part[3]}, peak {full[4] / 2 ** 30:.2f} -> {part[4] / 2 ** 30:.2f} GiB")
    assert part[3] < full[3] and part[4] < full[4]


def test_2x_loss_backward_heads_only():
    """`loss.backward()` on the 2x policy with only the heads training: the head gradients are the all-trainable ones bit for bit, every
    other .grad None."""
    pol = _policy("2x").set_autograd(True)
    img, first, actions = _frames(torch.Generator().manual_seed(3), 4)
    res = []
    for heads_only in (False, True):
        _unfreeze(pol)
        if heads_only:
            _freeze(pol, ("pi_head.",), keep=True)
        (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(4))
        loss = -pol.logprob(actions, pd).mean()
        loss.backward()
        nat.device_check()
        res.append((loss.detach(), {n: p.grad for n, p in pol.named_parameters()}))
        pol.zero_grad(set_to_none=True)
    (l0, g0), (l1, g1) = res
    assert torch.equal(l0, l1)
    for n in g1:
        if n.startswith("pi_head."):
            assert torch.equal(g1[n], g0[n]), n
        else:
            assert g1[n] is None, n
