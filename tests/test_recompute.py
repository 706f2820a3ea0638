"""`recompute_frames` (the trainers' constructors and `set_autograd`) on the CPU, through the test-only torch emulation of the ops: the forward
keeps only the ImpalaCNN's output and the backward re-runs the CNN chunk by chunk.  Checked against autograd through the oracle (bf16 rounding
off, several chunks per call) and against the stored-tape path bit for bit (bf16 rounding on, one chunk).  tests/test_gpu_recompute.py
repeats it through the CUDA kernels at the released model's shapes."""
import copy

import pytest
import torch

import emu_bptt_ops
import emu_rl_ops
import test_idm_training
import test_rl_training
import test_training
import vpt_oracle as O
from common import make_policy, small_kwargs
from test_autograd import _with_grad, batch, bc_loss, compare, emulated, exact, leaf_of  # noqa: F401  (fixtures)
from test_idm_training import make_batch, make_idm
from video_pre_training_b200 import ops
from video_pre_training_b200.training import BCTrainer, IDMTrainer, RLTrainer, _Trainer


@pytest.fixture()
def emu(emulated, monkeypatch):  # noqa: F811
    """The emulation of every op the BC, RL and IDM steps and the BPTT window use."""
    for name in dir(emu_rl_ops):
        if not name.startswith("_") and callable(getattr(emu_rl_ops, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(emu_rl_ops, name))
    monkeypatch.setattr(ops, "attention_bwd_state", _with_grad(emu_bptt_ops.attention_bwd_state))
    yield


def recomputing(cls, frames, chunks):
    """`cls` with recompute_frames=frames; every recomputed chunk's (f0, f1) goes to `chunks`."""
    class Recomputing(cls):
        def __init__(self, policy):
            super().__init__(policy, recompute_frames=frames)
            self.on_recompute = lambda f0, f1, out, mr: chunks.append((f0, f1))
    return Recomputing


def _grads(mod):
    return {n: None if p.grad is None else p.grad.clone() for n, p in mod.named_parameters()}


def assert_same_grads(a, b):
    assert a.keys() == b.keys()
    for n in a:
        assert (a[n] is None) == (b[n] is None), n
        if a[n] is not None:
            assert torch.equal(a[n], b[n]), (n, (a[n] - b[n]).abs().max().item())


def assert_same_state(sa, sb):
    for (ma, (ka, va)), (mb, (kb, vb)) in zip(sa, sb):
        assert (ma is None and mb is None) or torch.equal(ma, mb)
        assert torch.equal(ka, kb) and torch.equal(va, vb)


# ---------------------------------------------------------------------------------------------------------------
# several chunks per call: the exact gradient
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("step", ["bc", "rl", "idm"])
def test_recompute_in_chunks_is_the_exact_gradient(emu, exact, monkeypatch, step):
    """bf16 rounding off, 16 frames per call in CNN chunks of 8 (the IDM: one sequence per chunk): the trainers' own exact-gradient tests
    (two and three calls with carried state and an episode reset for BC, the clipped RL loss with the value head and the normaliser, the
    IDM loss with its conv3d pre-stage) pass unchanged with recompute_frames."""
    chunks = []
    if step == "bc":
        monkeypatch.setattr(test_training, "BCTrainer", recomputing(BCTrainer, 8, chunks))
        test_training.test_bc_backward_is_the_exact_gradient(None, None)
    elif step == "rl":
        monkeypatch.setattr(test_rl_training, "RLTrainer", recomputing(RLTrainer, 8, chunks))
        test_rl_training.test_rl_backward_is_the_exact_gradient(None, None)
    else:
        monkeypatch.setattr(test_idm_training, "IDMTrainer", recomputing(IDMTrainer, 8, chunks))
        test_idm_training.test_idm_backward_is_the_exact_gradient(None, None)
    assert chunks and set(chunks) == {(0, 8), (8, 16)}  # every call was two recomputed chunks, the last one first
    assert chunks[:2] == [(8, 16), (0, 8)]


def test_call_above_the_stored_limits_runs(emu, exact, monkeypatch):
    """With cnn_chunk_frames / idm_chunk_frames at 8 the stored tape refuses a call of 16 frames; with recompute_frames it runs (in CNN
    chunks of at most 8 frames, whatever recompute_frames says) and its gradient is the oracle's, through the trainers and through
    `loss.backward()`."""
    pol, sd, cfg = make_policy(small_kwargs())
    monkeypatch.setattr(pol.net, "cnn_chunk_frames", 8)
    g = torch.Generator().manual_seed(4)
    img, first, actions = batch(g, 2, 8, reset=(1, 5))
    with pytest.raises(NotImplementedError):
        BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
    assert all(p.grad is None for p in pol.parameters())
    tr = BCTrainer(pol, recompute_frames=2048)
    chunks = []
    tr.on_recompute = lambda f0, f1, out, mr: chunks.append((f0, f1))
    loss, _ = tr.loss_and_grad(img, first, pol.initial_state(2), actions)
    assert chunks == [(8, 16), (0, 8)]
    loss_o, grads_o, _ = test_training.oracle_grads(sd, cfg, img, first, O.initial_state(cfg, 2), actions)
    test_training.check([(loss, loss_o, _grads(pol), grads_o)])

    pol.zero_grad(set_to_none=True)
    pol.set_autograd(True, recompute_frames=8)
    (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(2))
    bc_loss(pol, pd, actions).backward()
    grads_o = {k: v for k, v in grads_o.items() if not k.startswith("value_head.")}
    assert compare({n: g_ for n, g_ in _grads(pol).items() if not n.startswith("value_head.")}, grads_o) > 40

    idm, sd, cfg = make_idm()
    monkeypatch.setattr(idm.net, "idm_chunk_frames", 8)
    img, first, actions = make_batch(g)
    with pytest.raises(NotImplementedError):
        IDMTrainer(idm).loss_and_grad(img, first, idm.initial_state(2), actions)
    tr = IDMTrainer(idm, recompute_frames=3)  # rounded to one sequence (8 frames)
    chunks = []
    tr.on_recompute = lambda f0, f1, out, mr: chunks.append((f0, f1))
    loss, _ = tr.loss_and_grad(img, first, idm.initial_state(2), actions)
    assert chunks == [(8, 16), (0, 8)]
    loss_o, grads_o = test_idm_training.oracle_grads(sd, cfg, img, first, actions)
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    for n, g_ in _grads(idm).items():
        test_idm_training.check_pattern(n, g_)
        if test_idm_training.kind(n) == "dense":
            cnn = n.startswith(("net.img_process.cnn.stacks", "net.conv3d_layer"))
            assert ((g_ - grads_o[n]).norm() / grads_o[n].norm()).item() < (5e-2 if cnn else 1e-3), n


def test_call_above_the_stored_limit_launches_nothing(emu, monkeypatch):
    """With cnn_chunk_frames at 8, a 16-frame BCTrainer or RLTrainer call on the stored tape raises before its first op: the CNN does not
    run (and tape) chunk after chunk first."""
    pol, _, _ = make_policy(small_kwargs())
    monkeypatch.setattr(pol.net, "cnn_chunk_frames", 8)
    launched = []
    for name in dir(ops):
        fn = getattr(ops, name)
        if not name.startswith("_") and callable(fn) and getattr(fn, "__module__", "").startswith(("emu_", "test_", "common")):
            monkeypatch.setattr(ops, name, lambda *a, _name=name, _fn=fn, **k: (launched.append(_name), _fn(*a, **k))[1])
    g = torch.Generator().manual_seed(5)
    img, first, actions = batch(g, 2, 8)
    z = torch.zeros(2, 8)
    with pytest.raises(NotImplementedError):
        BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
    with pytest.raises(NotImplementedError):
        RLTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions, z, z, z, vf_coef=0.5, kl_coef=0.0)
    assert launched == []
    assert all(p.grad is None for p in pol.parameters())
    BCTrainer(pol).loss_and_grad(img[:1], first[:1], pol.initial_state(1), actions_of(actions, 1))  # 8 frames: one chunk
    assert "conv3x3_zp" in launched


def test_bad_recompute_frames_and_the_call_limit(emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    idm, _, _ = make_idm(pert=False)
    for bad in (0, -8, 2.5, True, "8"):
        for make in (lambda: BCTrainer(pol, recompute_frames=bad), lambda: RLTrainer(pol, recompute_frames=bad),
                     lambda: IDMTrainer(idm, recompute_frames=bad), lambda: pol.set_autograd(True, recompute_frames=bad),
                     lambda: pol.net.set_autograd(True, recompute_frames=bad), lambda: idm.set_autograd(True, recompute_frames=bad)):
            with pytest.raises(ValueError):
                make()
    assert pol._recompute_frames is None and pol.net._recompute_frames is None
    assert pol.set_autograd(True, recompute_frames=64).net._recompute_frames == 64
    assert pol.set_autograd(False, recompute_frames=64)._recompute_frames is None  # off: nothing to recompute

    # the per-call frame limit is checked before any work: nothing reaches .grad
    monkeypatch.setattr(_Trainer, "max_call_frames", 15)
    g = torch.Generator().manual_seed(9)
    img, first, actions = batch(g, 2, 8)
    with pytest.raises(NotImplementedError):
        BCTrainer(pol, recompute_frames=8).loss_and_grad(img, first, pol.initial_state(2), actions)
    pol.set_autograd(True, recompute_frames=8)
    with pytest.raises(NotImplementedError):
        pol({"img": img}, first, pol.initial_state(2))
    assert all(p.grad is None for p in pol.parameters())
    BCTrainer(pol, recompute_frames=8).loss_and_grad(img[:1], first[:1], pol.initial_state(1), actions_of(actions, 1))
    monkeypatch.setattr(_Trainer, "max_call_batch", 1)
    with pytest.raises(NotImplementedError):
        BCTrainer(pol, recompute_frames=8).loss_and_grad(img[:, :4], first[:, :4], pol.initial_state(2), actions_of(actions, 2, 4))


def actions_of(actions, B, T=None):
    return {k: v[:B, :T] for k, v in actions.items()}


# ---------------------------------------------------------------------------------------------------------------
# one chunk: bit-identical to the stored tape, bf16 rounding on
# ---------------------------------------------------------------------------------------------------------------
def test_one_chunk_is_bit_identical_bc_and_rl(emu):
    """BCTrainer over two calls with carried state, and RLTrainer (the normaliser update and the statistics included): the loss, every
    `.grad` (None where the stored tape gives None) and state_out, bit for bit."""
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(1)
    batches = [batch(g, 2, 8, reset=(1, 2) if c else None) for c in range(2)]
    res = []
    for rf in (None, 16, 2048):
        pol = copy.deepcopy(pol0)
        tr = BCTrainer(pol, recompute_frames=rf)
        st, out = pol.initial_state(2), []
        for img, first, actions in batches:
            loss, st = tr.loss_and_grad(img, first, st, actions)
            out.append((loss, st, _grads(pol)))
        res.append(out)
    for out in res[1:]:
        for (l0, s0, g0), (l1, s1, g1) in zip(res[0], out):
            assert torch.equal(l0, l1)
            assert_same_state(s0, s1)
            assert_same_grads(g0, g1)

    pol0, sd, sd_ref, cfg = test_rl_training.make_pair()
    img, first, actions = batch(g, 2, 8, reset=(0, 3))
    pd_ref, _ = test_rl_training.ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, 2))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 2))
    old, adv, returns = test_rl_training.make_rl_batch(g, O.logprob(pd0, actions), 2, 8)
    res = []
    for rf in (None, 16):
        pol = copy.deepcopy(pol0)
        tr = RLTrainer(pol, recompute_frames=rf)
        loss, st = tr.loss_and_grad(img, first, pol.initial_state(2), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)
        norm = {k: getattr(pol.value_head.normalizer, k).clone() for k in test_rl_training.NORM}
        res.append((loss, st, _grads(pol), norm, {k: v.clone() for k, v in tr.stats.items()}))
    (l0, s0, g0, n0, t0), (l1, s1, g1, n1, t1) = res
    assert torch.equal(l0, l1)
    assert_same_state(s0, s1)
    assert_same_grads(g0, g1)
    assert g1["value_head.linear.weight"].abs().sum() > 0
    for k in n0:
        assert torch.equal(n0[k], n1[k]), k
    for k in t0:
        assert torch.equal(t0[k], t1[k]), k


def test_one_chunk_is_bit_identical_idm_and_autograd(emu):
    """IDMTrainer, `loss.backward()` on the agent policy and a two-call `state_grad` window with one backward: bit for bit."""
    idm0, _, _ = make_idm()
    g = torch.Generator().manual_seed(2)
    img, first, actions = make_batch(g)
    res = []
    for rf in (None, 16):
        idm = copy.deepcopy(idm0)
        loss, st = IDMTrainer(idm, recompute_frames=rf).loss_and_grad(img, first, idm.initial_state(2), actions)
        res.append((loss, st, _grads(idm)))
    assert torch.equal(res[0][0], res[1][0])
    assert_same_state(res[0][1], res[1][1])
    assert_same_grads(res[0][2], res[1][2])

    pol0, _, _ = make_policy(small_kwargs())
    batches = [batch(g, 2, 8, reset=(1, 6) if c else None) for c in range(2)]
    for state_grad in (False, True):
        res = []
        for rf in (None, 16):
            pol = copy.deepcopy(pol0).set_autograd(True, state_grad=state_grad, recompute_frames=rf)
            st, total, states = pol.initial_state(2), 0.0, []
            for img, first, actions in (batches if state_grad else batches[:1]):
                (pd, _, _), st = pol({"img": img}, first, st)
                total = total + bc_loss(pol, pd, actions)
                states.append([(m, (k.detach(), v.detach())) for m, (k, v) in st])
            total.backward()
            res.append((total.detach(), states, _grads(pol)))
        assert torch.equal(res[0][0], res[1][0])
        for s0, s1 in zip(res[0][1], res[1][1]):
            assert_same_state(s0, s1)
        assert_same_grads(res[0][2], res[1][2])
        assert res[1][2]["value_head.linear.weight"] is None


def test_recomputed_cnn_out_equals_the_stored_one(emu):
    """The backward's re-run of every chunk reproduces the forward's CNN output and statistics bit for bit (several chunks per call), and
    the forward records no per-stack activations."""
    pol, _, _ = make_policy(small_kwargs())
    idm, _, _ = make_idm()
    g = torch.Generator().manual_seed(3)
    cases = [(BCTrainer(pol, recompute_frames=5), batch(g, 2, 8), pol), (IDMTrainer(idm, recompute_frames=8), make_batch(g), idm)]
    for tr, (img, first, actions), mod in cases:
        tr.keep_tape = True
        seen = []
        tr.on_recompute = lambda f0, f1, out, mr: seen.append((f0, f1, out.clone(), mr.clone()))
        tr.loss_and_grad(img, first, mod.initial_state(2), actions)
        tape = tr.last_tape
        assert tape["stacks"] == [] and len(seen) == len(tape["cnn_chunks"]) >= 2
        assert sorted(s[:2] for s in seen) == tape["cnn_chunks"]
        for f0, f1, out, mr in seen:
            assert torch.equal(out, tape["cnn_out"][f0:f1])
            assert torch.equal(mr, tape["mr_c"][f0:f1])
    assert [c for c in cases[0][0].last_tape["cnn_chunks"]] == [(0, 5), (5, 10), (10, 15), (15, 16)]
