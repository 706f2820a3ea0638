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


def _same_latents(part, ref, label):
    nat.device_check()
    dx = (part.x.float() - ref.x.float()).abs().max().item()
    ds = (part.stats - ref.stats).abs().max().item()
    print(f"{label}: max |dx| {dx:.3e}, max |dstats| {ds:.3e}")
    assert torch.equal(part.x, ref.x) and torch.equal(part.stats, ref.stats), label


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
        _same_latents(mod.encode(frames[sl]), enc[sl], f"{type(mod).__name__} encode{sl} against the slice of the whole encoding")


@pytest.mark.parametrize("width", ["2x", "1x"])
def test_latents_of_a_few_frames_do_not_depend_on_the_encoded_batch(width):
    """A few frames take other launch plans in the CNN (narrow weight tiles, more pool blocks: other statistics partials) and in `dense`
    (the weight-streaming GEMM up to 8 rows); `encode` pads them to the count from which every plan is the full chunk's.  Every slice
    length from 1 frame to one past that count, against the same rows of a 2 x 48-frame encoding, and a call whose last 2048-frame chunk
    holds 2 frames (B = 2, T = 1025), whose frames copy two of its first chunk."""
    pol = _policy(width)
    g = torch.Generator().manual_seed(6)
    img = torch.randint(0, 256, (2, 48, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    whole = pol.encode(img)
    n = pol.net._batch_plan_frames(1)
    print(f"{width}: encode pads a chunk to {n} frames")
    assert 17 <= n < 48
    for L in range(1, n + 2):
        t0 = (5 * L) % (48 - L)
        _same_latents(pol.encode(img[1:2, t0:t0 + L]), whole[1:2, t0:t0 + L], f"{width} encode of {L} frames")
    long = torch.randint(0, 256, (2, 1025, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    long[1, 1023:1025] = long[0, 0:2]
    lat = pol.encode(long)
    _same_latents(lat[1, 1023:1025], lat[0, 0:2], f"{width} B=2 T=1025: the 2 frames of the last chunk against the same frames in the first")


def test_idm_latents_of_short_sequences_do_not_depend_on_the_encoded_batch():
    """The IDM re-batched along B at T = 8: every B of 1 .. 4 sequences against the rows of one 6 x 8 encoding (the IDM pads whole
    zero sequences)."""
    idm = _idm()
    img = torch.randint(0, 256, (6, 8, 128, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(7)).cuda()
    whole = idm.encode(img)
    for b0, b1 in ((0, 1), (3, 4), (1, 3), (2, 5), (5, 6)):
        _same_latents(idm.encode(img[b0:b1]), whole[b0:b1], f"IDM encode of B={b1 - b0} T=8 sequences")


def test_2x_frozen_cnn_step_of_four_frames_from_sliced_latents():
    """A frozen-CNN BC step at B = 1, T = 4 from latents sliced out of a 2 x 32-frame encoding: the step from the frames, bit for bit."""
    pol = _policy()
    _freeze_cnn(pol)
    img, _, actions = _frames(torch.Generator().manual_seed(8), 2, 32)
    lat = pol.encode(img)[1:2, 9:13]
    img, first = img[1:2, 9:13].contiguous(), torch.zeros(1, 4, dtype=torch.bool).cuda()
    actions = {k: a[1:2, 9:13].contiguous() for k, a in actions.items()}
    tr = BCTrainer(pol)
    _same(_step(pol, tr, lat, first, actions), _step(pol, tr, img, first, actions))
    print("2x frozen-CNN BC step B=1 T=4: from sliced latents == from frames, bit for bit")
