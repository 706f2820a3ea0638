"""Training and running the policies from cached CNN latents (`encode`, `FrameLatents`, `{"img_latent": ...}`) on the CPU, through the
test-only torch emulation of the ops: a call from `encode(img)` is the same call from `img` with the CNN part frozen, bit for bit, and runs
no CNN op; the calls that cannot be served raise before any op runs.  tests/test_gpu_latents.py repeats it through the CUDA kernels at the
released shapes."""
import copy

import pytest
import torch

import emu_dist_ops
import test_rl_training
import vpt_oracle as O
from common import make_policy, small_kwargs
from test_autograd import batch, bc_loss, emulated  # noqa: F401  (fixture)
from test_freeze import CNN_BWD_OPS, freeze
from test_idm_training import make_batch, make_idm
from test_recompute import _grads, assert_same_grads, assert_same_state, emu  # noqa: F401  (fixture)
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import FrameLatents
from video_pre_training_b200.training import BCTrainer, IDMTrainer, RLTrainer

# the CNN part's ops, forward and backward (the dense GEMMs are recognised by their weights, `OpRecorder.dense_gemms`)
CNN_OPS = {"conv3x3_zp", "firstconv_pool", "maxpool3s2", "conv3d_t5", "norm2_fold", "affine_norm_zp", "add_zp", "firstconv_dimg",
           "conv3d_t5_dimg"} | CNN_BWD_OPS


class OpRecorder:
    """Records every emulated op called through `ops` (name, args)."""

    def __init__(self, monkeypatch):
        self.calls = []
        for name in dir(ops):
            fn = getattr(ops, name)
            if not name.startswith("_") and callable(fn) and getattr(fn, "__module__", "").startswith(("emu_", "test_", "common")):
                monkeypatch.setattr(ops, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        def run(*args, **kwargs):
            self.calls.append((name, args))
            return fn(*args, **kwargs)
        return run

    def names(self):
        return {n for n, _ in self.calls}

    def dense_gemms(self, net):
        """GEMMs on the dense layer's forward or dgrad weights."""
        w = (net.prepared().dense[0], net.prepared_backward()["dense_t"])
        return [a for n, a in self.calls if n == "gemm" and len(a) > 1 and any(a[1] is x for x in w)]


def assert_no_cnn_op(rec, net):
    assert not CNN_OPS & rec.names(), CNN_OPS & rec.names()
    assert not rec.dense_gemms(net)


def assert_same_pd(a, b):
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


# ---------------------------------------------------------------------------------------------------------------
# a call from latents is the frozen-CNN call from frames, bit for bit, without a CNN op
# ---------------------------------------------------------------------------------------------------------------
def test_bc_from_latents_is_the_frozen_cnn_step(emu, monkeypatch):
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(1)
    batches = [batch(g, 2, 8, reset=(1, 2) if c else None) for c in range(2)]
    res = []
    for latents in (False, True):
        pol = copy.deepcopy(pol0)
        pre = freeze(pol, "cnn")
        lats = [pol.encode(img) for img, _, _ in batches] if latents else None
        tr, st, out = BCTrainer(pol, recompute_frames=8), pol.initial_state(2), []  # (recompute_frames: ignored from latents)
        tr.keep_tape = True
        rec = OpRecorder(monkeypatch) if latents else None
        for c, (img, first, actions) in enumerate(batches):
            loss, st = tr.loss_and_grad(lats[c] if latents else img, first, st, actions)
            out.append((loss, st))
        if latents:
            assert_no_cnn_op(rec, pol.net)
            tape = tr.last_tape
            assert "frames" not in tape and tape.get("cnn_out") is None and tape["cnn_chunks"] == [] and tape["stacks"] == []
        res.append((out, _grads(pol), pre, pol))
    (o0, g0, _, _), (o1, g1, pre, pol) = res
    for (l0, s0), (l1, s1) in zip(o0, o1):
        assert torch.equal(l0, l1)
        assert_same_state(s0, s1)
    assert_same_grads(g0, g1)
    for n, p in pol.named_parameters():  # frozen .grad as it was
        if n in pre:
            assert (p.grad is None) == (pre[n] is None) and (p.grad is None or torch.equal(p.grad, pre[n])), n


def test_rl_from_latents_is_the_frozen_cnn_step(emu, monkeypatch):
    """The RL step with the entropy bonus and the KL penalty; pd_ref from the reference policy's forward on the trained policy's latents
    (another network: accepted)."""
    monkeypatch.setattr(ops, "rl_head_bwd_ent", emu_dist_ops.rl_head_bwd_ent)
    pol0, sd, sd_ref, cfg = test_rl_training.make_pair()
    ref, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(2)
    img, first, actions = batch(g, 2, 8, reset=(0, 3))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 2))
    old, adv, returns = test_rl_training.make_rl_batch(g, O.logprob(pd0, actions), 2, 8)
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref.initial_state(2))
    res = []
    for latents in (False, True):
        pol = copy.deepcopy(pol0)
        freeze(pol, "cnn")
        x = pol.encode(img) if latents else img
        rec = OpRecorder(monkeypatch) if latents else None
        if latents:
            with torch.no_grad():
                (pd_ref_lat, _, _), _ = ref({"img_latent": x}, first, ref.initial_state(2))
        tr = RLTrainer(pol)
        loss, st = tr.loss_and_grad(x, first, pol.initial_state(2), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1,
                                    ent_coef=0.01)
        if latents:
            assert_no_cnn_op(rec, pol.net)
            assert_no_cnn_op(rec, ref.net)
        norm = {k: getattr(pol.value_head.normalizer, k).clone() for k in test_rl_training.NORM}
        res.append((loss, st, _grads(pol), norm, dict(tr.stats)))
    (l0, s0, g0, n0, t0), (l1, s1, g1, n1, t1) = res
    assert torch.equal(l0, l1)
    assert_same_state(s0, s1)
    assert_same_grads(g0, g1)
    assert t0.keys() == t1.keys() and "entropy" in t0
    for d0, d1 in ((n0, n1), (t0, t1)):
        for k in d0:
            assert torch.equal(d0[k], d1[k]), k
    # the reference policy from latents: its upper part on the training layout's CNN output, within the bf16 tolerance of its frames path
    for k in pd_ref:
        assert (pd_ref[k] - pd_ref_lat[k]).abs().max().item() < 5e-2, k


def test_idm_from_latents_is_the_frozen_cnn_step(emu, monkeypatch):
    idm0, _, _ = make_idm()
    g = torch.Generator().manual_seed(3)
    img, first, actions = make_batch(g)
    res = []
    for latents in (False, True):
        idm = copy.deepcopy(idm0)
        freeze(idm, "cnn")
        x = idm.encode(img) if latents else img
        rec = OpRecorder(monkeypatch) if latents else None
        loss, st = IDMTrainer(idm).loss_and_grad(x, first, idm.initial_state(2), actions)
        if latents:
            assert_no_cnn_op(rec, idm.net)
        res.append((loss, st, _grads(idm)))
    (l0, s0, g0), (l1, s1, g1) = res
    assert torch.equal(l0, l1)
    assert_same_state(s0, s1)
    assert_same_grads(g0, g1)


@pytest.mark.parametrize("state_grad", [False, True])
def test_loss_backward_from_latents_is_the_frozen_cnn_call(emu, monkeypatch, state_grad):
    """`loss.backward()` over one call, and with state_grad over a two-call window with one backward: pd, vpred, state_out, the loss and
    every trainable .grad bit for bit."""
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(4)
    batches = [batch(g, 2, 8, reset=(1, 6) if c else None) for c in range(2)]
    res = []
    for latents in (False, True):
        pol = copy.deepcopy(pol0).set_autograd(True, state_grad=state_grad, recompute_frames=8)
        freeze(pol, "cnn")
        lats = [pol.encode(img) for img, _, _ in batches] if latents else None
        rec = OpRecorder(monkeypatch) if latents else None
        st, total, outs = pol.initial_state(2), 0.0, []
        for c, (img, first, actions) in enumerate(batches if state_grad else batches[:1]):
            (pd, vpred, _), st = pol({"img_latent": lats[c]} if latents else {"img": img}, first, st)
            total = total + bc_loss(pol, pd, actions) + 0.1 * (vpred ** 2).mean()
            outs.append(({k: v.detach() for k, v in pd.items()}, vpred.detach(), [(m, (k.detach(), v.detach())) for m, (k, v) in st]))
        total.backward()
        if latents:
            assert_no_cnn_op(rec, pol.net)
        res.append((total.detach(), outs, _grads(pol)))
    (l0, o0, g0), (l1, o1, g1) = res
    assert torch.equal(l0, l1)
    for (pd0, v0, s0), (pd1, v1, s1) in zip(o0, o1):
        assert torch.equal(v0, v1)
        assert_same_pd(pd0, pd1)
        assert_same_state(s0, s1)
    assert_same_grads(g0, g1)


def test_inference_from_latents_is_the_taped_forward(emu):
    """`{"img_latent": ...}` under no_grad: the agent, `get_output_for_observation`, the bare network, the IDM and `predict` give the taped
    forward's outputs from the same latents bit for bit."""
    pol, _, _ = make_policy(small_kwargs())
    freeze(pol, "cnn", preset=False)
    img, first, actions = batch(torch.Generator().manual_seed(5), 2, 8, reset=(1, 2))
    lat = pol.encode(img)
    tr = BCTrainer(pol)
    _, pd_t, v_t, _, st_t = tr._taped_forward(lat, first, pol.initial_state(2))
    with torch.no_grad():
        (pd, v, _), st = pol({"img_latent": lat}, first, pol.initial_state(2))
        lat_net, st_n = pol.net({"img_latent": lat}, pol.initial_state(2), {"first": first})
        pd1, v1, _ = pol.get_output_for_observation({"img_latent": lat[:, 0]}, pol.initial_state(2), first[:, 0])
    assert_same_pd(pd, pd_t)
    assert torch.equal(v, v_t)
    assert_same_state(st, st_t)
    assert_same_state(st_n, st_t)
    assert torch.equal(lat_net[0], tr._taped_latent(lat, first, pol.initial_state(2))[1])
    _, pd_t1, v_t1, _, _ = tr._taped_forward(lat[:, :1], first[:, :1], pol.initial_state(2))
    assert_same_pd(pd1, pd_t1)
    assert torch.equal(v1, pol.denormalize(v_t1)[:, 0])

    idm, _, _ = make_idm()
    img, first, _ = make_batch(torch.Generator().manual_seed(6))
    lat = idm.encode(img)
    _, pd_t, _, _, _ = IDMTrainer(idm)._taped_forward(lat, first, idm.initial_state(2))
    ac, _, res = idm.predict({"img_latent": lat}, first=first, state_in=idm.initial_state(2))
    assert_same_pd(res["pd"], pd_t)


# ---------------------------------------------------------------------------------------------------------------
# refused before any op runs
# ---------------------------------------------------------------------------------------------------------------
def _refused(monkeypatch, mod, call, match):
    before = {n: None if p.grad is None else p.grad.clone() for n, p in mod.named_parameters()}
    rec = OpRecorder(monkeypatch)
    with pytest.raises(ValueError, match=match):
        call()
    assert rec.calls == []
    for n, p in mod.named_parameters():
        assert (p.grad is None) == (before[n] is None) and (p.grad is None or torch.equal(p.grad, before[n])), n


def test_calls_that_cannot_be_served_raise_before_any_op(emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    img, first, actions = batch(torch.Generator().manual_seed(7), 2, 8)
    lat = pol.encode(img)
    freeze(pol, "cnn")  # (preset .grad on some frozen parameters: must survive)
    params = dict(pol.named_parameters())
    bc = lambda x: BCTrainer(pol).loss_and_grad(x, first, pol.initial_state(2), actions)  # noqa: E731
    fwd = lambda x: pol.set_autograd(True)({"img_latent": x}, first, pol.initial_state(2))  # noqa: E731
    for name in ("net.img_process.cnn.stacks.1.blocks.0.conv1.layer.weight", "net.img_process.cnn.dense.norm.bias"):
        params[name].requires_grad_(True)
        for call in (bc, fwd):
            _refused(monkeypatch, pol, lambda: call(lat), name[4:])
        params[name].requires_grad_(False)
    # an image gradient through latents
    lg = FrameLatents(lat.x.clone(), lat.stats, lat.token)
    lg.x.requires_grad_(True)
    for call in (bc, fwd):
        _refused(monkeypatch, pol, lambda: call(lg), "no autograd graph")
    with pytest.raises(ValueError):
        FrameLatents(lg.x, lat.stats)
    # a cnn_outsize mismatch
    narrow = FrameLatents(lat.x[..., :128].contiguous(), lat.stats, lat.token)
    for call in (bc, fwd):
        _refused(monkeypatch, pol, lambda: call(narrow), "latents must be")
    pol.set_autograd(False)
    with torch.no_grad():
        _refused(monkeypatch, pol, lambda: pol({"img_latent": narrow}, first, pol.initial_state(2)), "latents must be")
    # stale: the encoding network's CNN changed since; another network (a copy) takes them
    other = copy.deepcopy(pol)
    with torch.no_grad():
        params["net.img_process.cnn.stacks.0.n.weight"].mul_(1.0)  # an in-place update
    for call in (bc, fwd):
        _refused(monkeypatch, pol, lambda: call(lat), "stale")
    pol.set_autograd(False)
    with torch.no_grad():
        _refused(monkeypatch, pol, lambda: pol({"img_latent": lat}, first, pol.initial_state(2)), "stale")
        other({"img_latent": lat}, first, other.initial_state(2))
    BCTrainer(other).loss_and_grad(lat, first, other.initial_state(2), actions)

    idm, _, _ = make_idm()
    img, first, actions = make_batch(torch.Generator().manual_seed(8))
    lat = idm.encode(img)
    freeze(idm, "cnn")
    w3 = idm.net.conv3d_layer.layer.weight
    w3.requires_grad_(True)
    _refused(monkeypatch, idm, lambda: IDMTrainer(idm).loss_and_grad(lat, first, idm.initial_state(2), actions), "conv3d_layer")
    w3.requires_grad_(False)
    IDMTrainer(idm).loss_and_grad(lat, first, idm.initial_state(2), actions)


def test_encode_runs_in_the_bf16_mode_only(emu):
    pol, _, _ = make_policy(small_kwargs())
    img, _, _ = batch(torch.Generator().manual_seed(9), 1, 2)
    pol.set_precision("fp32")
    with pytest.raises(NotImplementedError):
        pol.encode(img)


# ---------------------------------------------------------------------------------------------------------------
# batching latents
# ---------------------------------------------------------------------------------------------------------------
def _same_lat(a, b):
    assert torch.equal(a.x, b.x) and torch.equal(a.stats, b.stats)


def test_indexing_and_cat_give_the_encoding_of_those_frames(emu):
    pol, _, _ = make_policy(small_kwargs())
    img, _, _ = batch(torch.Generator().manual_seed(10), 4, 8)
    lat = pol.encode(img)
    assert tuple(lat.shape) == (4, 8) and lat.x.dtype == torch.bfloat16 and lat.stats.shape == (4, 8, 2)
    _same_lat(lat[1:3], pol.encode(img[1:3]))
    _same_lat(lat[:, 2:6], pol.encode(img[:, 2:6]))
    _same_lat(lat[torch.tensor([3, 0])], pol.encode(img[torch.tensor([3, 0])]))
    _same_lat(FrameLatents.cat([lat[2:], lat[:2]], 0), pol.encode(torch.cat([img[2:], img[:2]], 0)))
    _same_lat(FrameLatents.cat([lat[:, :3], lat[:, 3:]], dim=-1), lat)
    _same_lat(lat.to("cpu"), lat)
    assert lat[0, 1].x.shape == (256,) and lat[:, None].shape == (4, 1, 8)
    for bad in ((Ellipsis, 0), (0, 0, 0)):
        with pytest.raises(IndexError):
            lat[bad]
    with pytest.raises(IndexError):
        FrameLatents.cat([lat, lat], 2)
    other, _, _ = make_policy(small_kwargs())
    with pytest.raises(ValueError):
        FrameLatents.cat([lat, other.encode(img)], 0)

    idm, _, _ = make_idm()
    img, _, _ = make_batch(torch.Generator().manual_seed(11), B=3)
    lat = idm.encode(img)
    _same_lat(lat[1:], idm.encode(img[1:]))  # re-batched along B (not along T: the conv3d pre-stage mixes neighbouring frames)
    _same_lat(FrameLatents.cat([lat[2:], lat[:1]], 0), idm.encode(img[torch.tensor([2, 0])]))
