"""Training and running the policies from cached CNN latents on the H100 at the released models' shapes: a step from `encode(img)` is the
frozen-CNN step from `img` bit for bit, and faster; a 16384-frame call from latents needs no `recompute_frames`; `{"img_latent": ...}`
inference is the taped forward from the same latents bit for bit and within the 1e-2 tolerance of the frames path; a frame's latent does
not depend on the batch it was encoded in.  tests/test_latents.py checks the same rules on the CPU emulation."""
import pytest
import torch

import vpt_b200
from common import perturb
from video_pre_training_b200 import _native as nat
from video_pre_training_b200.training import BCTrainer, IDMTrainer

pytestmark = pytest.mark.gpu


def _policy(width="2x"):
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS)
    perturb(pol)
    return pol.cuda()


def _idm():
    torch.manual_seed(0)
    return vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()


def _frames(g, B, T=128):
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    return img, torch.zeros(B, T, dtype=torch.bool).cuda(), actions


def _freeze_cnn(mod):
    for n, p in mod.named_parameters():
        if n.startswith(("net.img_process.cnn.", "net.conv3d_layer.")):
            p.requires_grad_(False)


def _step(mod, tr, x, first, actions):
    """One call -> (loss, state_out, {name: .grad} (moved out), ms)."""
    for p in mod.parameters():
        p.grad = None
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    loss, st = tr.loss_and_grad(x, first, mod.initial_state(first.shape[0]), actions)
    e1.record()
    torch.cuda.synchronize()
    nat.device_check()
    grads = {}
    for n, p in mod.named_parameters():
        grads[n], p.grad = p.grad, None
    return loss, st, grads, e0.elapsed_time(e1)


def _same(a, b):
    (l0, s0, g0, _), (l1, s1, g1, _) = a, b
    assert torch.equal(l0, l1)
    for (_, (k0, v0)), (_, (k1, v1)) in zip(s0, s1):
        assert torch.equal(k0, k1) and torch.equal(v0, v1)
    assert g0.keys() == g1.keys()
    for n in g0:
        assert (g0[n] is None) == (g1[n] is None), n
        assert g0[n] is None or torch.equal(g0[n], g1[n]), n


def _compare(mod, tr, img, first, actions, label):
    """The frozen-CNN step from frames against the step from `encode(img)`, alternating (the first round warms up): bit-identical results,
    and the latent step is faster (medians)."""
    lat = mod.encode(img)
    times = ([], [])
    for r in range(4):
        frames_run = _step(mod, tr, img, first, actions)
        lat_run = _step(mod, tr, lat, first, actions)
        _same(lat_run, frames_run)
        if r:
            times[0].append(frames_run[3])
            times[1].append(lat_run[3])
    med = [sorted(t)[len(t) // 2] for t in times]
    print(f"{label}: frozen CNN from frames {med[0]:.1f} ms, from latents {med[1]:.1f} ms")
    assert med[1] < med[0]


def test_2x_bc_from_latents_is_the_frozen_cnn_step_and_faster():
    pol = _policy()
    _freeze_cnn(pol)
    img, first, actions = _frames(torch.Generator().manual_seed(0), 16)
    _compare(pol, BCTrainer(pol), img, first, actions, "2x BC B=16 T=128")


def test_4x_idm_from_latents_is_the_frozen_cnn_step_and_faster():
    idm = _idm()
    _freeze_cnn(idm)
    g = torch.Generator().manual_seed(1)
    img = torch.randint(0, 256, (4, 128, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(4, 128, dtype=torch.bool).cuda()
    actions = {"buttons": torch.randint(0, 2, (4, 128, 20), generator=g).cuda(), "camera": torch.randint(0, 11, (4, 128, 2), generator=g).cuda()}
    _compare(idm, IDMTrainer(idm), img, first, actions, "4x IDM B=4 T=128")


def test_2x_bc_16384_frames_from_latents_in_one_call():
    """B = 128, T = 128 in one call from latents without recompute_frames: the frozen-CNN call from frames, bit for bit."""
    pol = _policy()
    _freeze_cnn(pol)
    img, first, actions = _frames(torch.Generator().manual_seed(2), 128)
    tr = BCTrainer(pol)
    lat = pol.encode(img)
    torch.cuda.reset_peak_memory_stats()
    lat_run = _step(pol, tr, lat, first, actions)
    peak = torch.cuda.max_memory_allocated()
    frames_run = _step(pol, tr, img, first, actions)
    _same(lat_run, frames_run)
    print(f"2x BC B=128 T=128 from latents: {lat_run[3]:.1f} ms, peak {peak / 2 ** 30:.2f} GiB")


def test_inference_from_latents():
    """`{"img_latent": ...}` under no_grad: the taped forward from the same latents bit for bit, and within 1e-2 of the frames path."""
    pol = _policy()
    _freeze_cnn(pol)
    img, first, _ = _frames(torch.Generator().manual_seed(3), 4)
    lat = pol.encode(img)
    with torch.no_grad():
        (pd, v, _), st = pol({"img_latent": lat}, first, pol.initial_state(4))
        (pd_f, v_f, _), _ = pol({"img": img}, first, pol.initial_state(4))
    _, pd_t, v_t, _, st_t = BCTrainer(pol)._taped_forward(lat, first, pol.initial_state(4))
    nat.device_check()
    assert torch.equal(v, v_t)
    for k in pd:
        assert torch.equal(pd[k], pd_t[k]), k
        err = ((pd[k] - pd_f[k]).abs() / pd_f[k].abs()).max().item()
        print(f"2x inference from latents vs frames: {k} max rel err {err:.2e}")
        assert err < 1e-2, (k, err)
    for (_, (k0, v0)), (_, (k1, v1)) in zip(st, st_t):
        assert torch.equal(k0, k1) and torch.equal(v0, v1)


def test_latent_rows_do_not_depend_on_the_encoded_batch():
    """`encode` of a slice against the slice of a whole encoding: the 2x agent over B = 16 against B = 3 and 5 (rows of frames the
    convolution tiles differently), the 4x IDM over B = 4 against B = 1 (re-batched along B only)."""
    pol = _policy()
    img, _, _ = _frames(torch.Generator().manual_seed(4), 16)
    whole = pol.encode(img)
    cases = [(pol, img, whole, sl) for sl in ((slice(0, 3),), (slice(7, 12),), (slice(15, 16),), (slice(2, 3), slice(5, 38)))]
    idm = _idm()
    img_i = torch.randint(0, 256, (4, 128, 128, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).cuda()
    cases.append((idm, img_i, idm.encode(img_i), (slice(2, 3),)))
    for mod, frames, enc, sl in cases:
        part, ref = mod.encode(frames[sl]), enc[sl]
        nat.device_check()
        dx = (part.x.float() - ref.x.float()).abs().max().item()
        ds = (part.stats - ref.stats).abs().max().item()
        print(f"{type(mod).__name__} encode{sl} against the slice of the whole encoding: max |dx| {dx:.3e}, max |dstats| {ds:.3e}")
        assert torch.equal(part.x, ref.x) and torch.equal(part.stats, ref.stats), sl
