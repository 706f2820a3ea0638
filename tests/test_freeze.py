"""Training part of a policy (`requires_grad_(False)` on some parameters) on the CPU, through the test-only torch emulation of the ops: a
frozen parameter gets no gradient, the trainable ones get exactly the gradient of the all-trainable step, and the work that only served
frozen parameters (their weight-side sums, the input gradients below the lowest trainable unit, the CNN tape) is not done.
tests/test_gpu_freeze.py repeats it through the CUDA kernels at the released shapes."""
import copy

import pytest
import torch

import test_rl_training
import vpt_oracle as O
from common import make_policy, small_kwargs
from test_autograd import batch, bc_loss, compare, emulated, exact  # noqa: F401  (fixtures)
from test_idm_training import check_pattern, kind, make_batch, make_idm
from test_recompute import _grads, assert_same_state, emu  # noqa: F401  (fixture)
from video_pre_training_b200 import ops
from video_pre_training_b200.training import BCTrainer, IDMTrainer, RLTrainer

PATTERNS = {
    "cnn": ("img_process.cnn.", "conv3d_layer."),                      # (a) the CNN (the IDM: with its conv3d pre-stage)
    "below_transformer": ("img_process.", "conv3d_layer."),           # (b) everything below the transformer
    "stacks01": ("img_process.cnn.stacks.0.", "img_process.cnn.stacks.1."),  # (c) the lower two stacks
    "blocks01": ("recurrent_layer.blocks.0.", "recurrent_layer.blocks.1."),  # (d) two transformer blocks, the CNN training
    "norms": None,                                                    # (e) every norm affine
    "heads_only": "heads",                                            # (f) all but the heads
}
CNN_BWD_OPS = {"conv3x3_zp", "affine_norm_zp", "norm_sums", "maxpool3s2_bwd", "firstconv_bwd", "conv3d_t5_bwd", "add_zp"}


def frozen(name, pattern):
    """Whether parameter `name` (without the policy's "net." prefix for network parameters) is frozen under `pattern`."""
    n = name[4:] if name.startswith("net.") else name
    spec = PATTERNS.get(pattern, pattern)
    if spec is None:
        return ".norm." in n or "_ln." in n or ".n." in n
    if spec == "heads":
        return not n.startswith("pi_head.")
    if spec == "value_head":
        return not n.startswith("value_head.")
    return n.startswith(spec)


def freeze(mod, pattern, preset=True):
    """requires_grad_(False) on the parameters `pattern` names; every other frozen parameter gets a `.grad` set beforehand (which must
    survive the call).  -> {name: preset gradient or None} of the frozen parameters."""
    pre = {}
    for i, (n, p) in enumerate(mod.named_parameters()):
        if p.requires_grad and frozen(n, pattern):
            p.requires_grad_(False)
            p.grad = torch.full_like(p, 0.5 + i) if preset and i % 2 else None
            pre[n] = None if p.grad is None else p.grad.clone()
    assert pre
    return pre


def check_partial(grads_all, mod, pre):
    """Every trainable parameter's .grad equals the all-trainable run's bit for bit; every frozen .grad is as it was before the call."""
    for n, p in mod.named_parameters():
        if n in pre:
            assert (p.grad is None) == (pre[n] is None) and (p.grad is None or torch.equal(p.grad, pre[n])), n
        elif grads_all[n] is None:
            assert p.grad is None, n
        else:
            assert p.grad is not None and torch.equal(p.grad, grads_all[n]), (n, (p.grad - grads_all[n]).abs().max().item())


class OpLog:
    """Records the emulated ops the backward runs (from the first `_heads_bwd` / `_backward_from_dlat` of a trainer on)."""

    def __init__(self, monkeypatch, tr):
        self.calls, self.bwd = [], False
        for name in dir(ops):
            fn = getattr(ops, name)
            if not name.startswith("_") and callable(fn) and getattr(fn, "__module__", "").startswith(("emu_", "test_", "common")):
                monkeypatch.setattr(ops, name, self._wrap(name, fn))
        for meth in ("_heads_bwd", "_backward_from_dlat"):
            monkeypatch.setattr(tr, meth, self._enter(getattr(tr, meth)))

    def _wrap(self, name, fn):
        def run(*args, **kwargs):
            self.calls.append((self.bwd, name, args))
            return fn(*args, **kwargs)
        return run

    def _enter(self, fn):
        def run(*args, **kwargs):
            self.bwd = True
            return fn(*args, **kwargs)
        return run

    def names(self, bwd=True):
        return [n for b, n, _ in self.calls if b == bwd]

    def reads(self, x, names):
        """Whether a backward op in `names` took tensor x as an argument."""
        return any(b and n in names and any(a is x for a in args) for b, n, args in self.calls)


# ---------------------------------------------------------------------------------------------------------------
# bit-identical trainable gradients, bf16 rounding on
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_bc_trainer_trains_part_bit_identically(emu, pattern):
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(1)
    batches = [batch(g, 2, 8, reset=(1, 2) if c else None) for c in range(2)]
    res = []
    for part in (False, True):
        pol = copy.deepcopy(pol0)
        pre = freeze(pol, pattern) if part else None
        tr, st, out = BCTrainer(pol), pol.initial_state(2), []
        for img, first, actions in batches:
            loss, st = tr.loss_and_grad(img, first, st, actions)
            out.append((loss, st))
        res.append((out, pol, pre))
    (out0, pol_all, _), (out1, pol, pre) = res
    for (l0, s0), (l1, s1) in zip(out0, out1):
        assert torch.equal(l0, l1)
        assert_same_state(s0, s1)
    check_partial(_grads(pol_all), pol, pre)


@pytest.mark.parametrize("pattern", ["cnn", "blocks01", "norms", "heads_only", "value_head"])
def test_rl_trainer_trains_part_bit_identically(emu, pattern):
    pol0, sd, sd_ref, cfg = test_rl_training.make_pair()
    g = torch.Generator().manual_seed(2)
    img, first, actions = batch(g, 2, 8, reset=(0, 3))
    pd_ref, _ = test_rl_training.ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, 2))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 2))
    old, adv, returns = test_rl_training.make_rl_batch(g, O.logprob(pd0, actions), 2, 8)
    res = []
    for part in (False, True):
        pol = copy.deepcopy(pol0)
        pre = freeze(pol, pattern) if part else None
        tr = RLTrainer(pol)
        loss, st = tr.loss_and_grad(img, first, pol.initial_state(2), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)
        norm = {k: getattr(pol.value_head.normalizer, k).clone() for k in test_rl_training.NORM}
        res.append((loss, st, pol, pre, norm, dict(tr.stats)))
    (l0, s0, pol_all, _, n0, t0), (l1, s1, pol, pre, n1, t1) = res
    assert torch.equal(l0, l1)
    assert_same_state(s0, s1)
    check_partial(_grads(pol_all), pol, pre)
    for k in n0:
        assert torch.equal(n0[k], n1[k]), k
    for k in t0:
        assert torch.equal(t0[k], t1[k]), k
    if pattern == "value_head":
        assert pol.value_head.linear.weight.grad.abs().sum() > 0


@pytest.mark.parametrize("pattern", ["cnn", "below_transformer", "stacks01", "norms", "heads_only"])
def test_idm_trainer_trains_part_bit_identically(emu, pattern):
    idm0, _, _ = make_idm()
    g = torch.Generator().manual_seed(3)
    img, first, actions = make_batch(g)
    res = []
    for part in (False, True):
        idm = copy.deepcopy(idm0)
        pre = freeze(idm, pattern) if part else None
        loss, st = IDMTrainer(idm).loss_and_grad(img, first, idm.initial_state(2), actions)
        res.append((loss, st, idm, pre))
    (l0, s0, idm_all, _), (l1, s1, idm, pre) = res
    assert torch.equal(l0, l1)
    assert_same_state(s0, s1)
    check_partial(_grads(idm_all), idm, pre)


@pytest.mark.parametrize("pattern", ["cnn", "below_transformer", "stacks01", "blocks01", "norms", "heads_only"])
@pytest.mark.parametrize("state_grad", [False, True])
def test_loss_backward_trains_part_bit_identically(emu, pattern, state_grad):
    """`loss.backward()` over one call, and with state_grad over a two-call window with one backward: pd, vpred, state_out, the loss and
    every trainable .grad bit for bit; frozen .grad untouched."""
    pol0, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(4)
    batches = [batch(g, 2, 8, reset=(1, 6) if c else None) for c in range(2)]
    res = []
    for part in (False, True):
        pol = copy.deepcopy(pol0).set_autograd(True, state_grad=state_grad)
        pre = freeze(pol, pattern) if part else None
        st, total, outs = pol.initial_state(2), 0.0, []
        for img, first, actions in (batches if state_grad else batches[:1]):
            (pd, vpred, _), st = pol({"img": img}, first, st)
            total = total + bc_loss(pol, pd, actions) + 0.1 * (vpred ** 2).mean()
            outs.append(({k: v.detach() for k, v in pd.items()}, vpred.detach(), [(m, (k.detach(), v.detach())) for m, (k, v) in st]))
        total.backward()
        res.append((total.detach(), outs, pol, pre))
    (l0, o0, pol_all, _), (l1, o1, pol, pre) = res
    assert torch.equal(l0, l1)
    for (pd0, v0, s0), (pd1, v1, s1) in zip(o0, o1):
        assert torch.equal(v0, v1) and all(torch.equal(pd0[k], pd1[k]) for k in pd0)
        assert_same_state(s0, s1)
    check_partial(_grads(pol_all), pol, pre)


# ---------------------------------------------------------------------------------------------------------------
# oracle parity, bf16 rounding off
# ---------------------------------------------------------------------------------------------------------------
def oracle_leaf(sd, pattern):
    return {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.") and not frozen(k, pattern))
            for k, v in sd.items()}


@pytest.mark.parametrize("pattern", ["cnn", "stacks01", "blocks01", "norms", "heads_only"])
def test_partial_gradient_is_the_oracles(emu, exact, pattern):
    """BCTrainer and `loss.backward()` against autograd through the oracle with the same requires_grad flags: the same parameters get
    None, the others the oracle's gradient.  (The batches are those of test_autograd's exact-gradient tests: on some batches a ReLU mask
    that sits at zero flips between the emulation and the oracle and moves a gradient by more than the tolerance, freezing or not.)"""
    pol0, sd, cfg = make_policy(small_kwargs())
    img, first, actions = batch(torch.Generator().manual_seed(0), 2, 8)
    # torch's CPU group_norm backward (2.11) crashes on a channels-last input that needs no gradient when its affine does: stack 2's first
    # norm with stacks 0-1 frozen.  There the oracle runs with every leaf trainable and drops the frozen leaves' gradients (whether a leaf
    # requires grad does not change the others' gradients).
    via_all = pattern == "stacks01"
    leaf = oracle_leaf(sd, "heads_only" if via_all else pattern)
    if via_all:
        leaf = {k: v.detach().requires_grad_(True) if v.dtype.is_floating_point and not k.startswith("value_head.normalizer.") else v
                for k, v in leaf.items()}
    (pd_o, _, _), _ = O.agent_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    (-O.logprob(pd_o, actions).mean()).backward()
    grads_o = {k: None if frozen(k, pattern) else v.grad for k, v in leaf.items()}
    for autograd in (False, True):
        pol = copy.deepcopy(pol0)
        freeze(pol, pattern, preset=False)
        if autograd:
            (pd, _, _), _ = pol.set_autograd(True)({"img": img}, first, pol.initial_state(2))
            bc_loss(pol, pd, actions).backward()
        else:
            BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
        compare(_grads(pol), grads_o)

    idm0, sd, cfg = make_idm()
    img, first, actions = make_batch(torch.Generator().manual_seed(0))
    leaf = oracle_leaf(sd, pattern)
    if via_all:
        leaf = {k: v.detach().requires_grad_(v.dtype.is_floating_point) for k, v in leaf.items()}
    (pd_o, _, _), _ = O.idm_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    (-O.logprob(pd_o, actions).mean()).backward()
    idm = copy.deepcopy(idm0)
    freeze(idm, pattern, preset=False)
    IDMTrainer(idm).loss_and_grad(img, first, idm.initial_state(2), actions)
    grads = _grads(idm)
    special = {n for n in grads if kind(n) != "dense"}
    for n in special:  # lastlayer None, r_layer zeros, b_nd empty when they train (IDMTrainer's pattern); None when frozen
        if frozen(n, pattern):
            assert grads[n] is None, n
        else:
            check_pattern(n, grads[n])
    compare({n: v for n, v in grads.items() if n not in special}, {n: None if frozen(n, pattern) else v.grad for n, v in leaf.items() if n not in special})


# ---------------------------------------------------------------------------------------------------------------
# work skipped
# ---------------------------------------------------------------------------------------------------------------
def test_frozen_cnn_runs_no_cnn_backward(emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    freeze(pol, "cnn")
    g = torch.Generator().manual_seed(6)
    img, first, actions = batch(g, 2, 8)
    for rf in (None, 8):
        tr = BCTrainer(pol, recompute_frames=rf)
        tr.keep_tape = True
        seen = []
        tr.on_recompute = lambda *a: seen.append(a)
        log = OpLog(monkeypatch, tr)
        tr.loss_and_grad(img, first, pol.initial_state(2), actions)
        assert not CNN_BWD_OPS & set(log.names()) and not seen
        assert "gemm" in log.names() and "norm_bwd_apply" in log.names()
        tape = tr.last_tape
        assert tape["stacks"] == [] and tape["cnn_chunks"] == [] and tape["cnn_out"] is None
        assert not log.reads(tape["xd"], {"group_sums", "norm_bwd_apply"})  # img_process.linear is the lowest unit: no d xd


def test_heads_only_runs_the_heads_backward_alone(emu, monkeypatch):
    pol, _, _ = make_policy(small_kwargs())
    freeze(pol, "heads_only")
    g = torch.Generator().manual_seed(7)
    img, first, actions = batch(g, 2, 8)
    tr = BCTrainer(pol)
    tr.keep_tape = True
    log = OpLog(monkeypatch, tr)
    called = []
    monkeypatch.setattr(tr, "_backward_from_dlat", lambda *a, **k: called.append(1))
    ugr = []
    tr.loss_and_grad(img, first, pol.initial_state(2), actions, upper_grads_ready=lambda: ugr.append(1))
    assert sorted(set(log.names())) == ["col_sums", "wgrad"] and not called and ugr == [1]
    assert all(b is None for b in tr.last_tape["blocks"])


def test_lowest_trainable_unit_gets_no_input_gradient(emu, monkeypatch):
    """Everything below the transformer frozen: block 0's pre_r_ln trains but its input gradient is not computed.  Stacks 0-1 frozen:
    stack 2's first conv trains, stacks 0-1 record nothing, and only stack 2's max-pool backward runs."""
    pol, _, _ = make_policy(small_kwargs())
    freeze(pol, "below_transformer")
    g = torch.Generator().manual_seed(8)
    img, first, actions = batch(g, 2, 8)
    tr = BCTrainer(pol)
    tr.keep_tape = True
    log = OpLog(monkeypatch, tr)
    ugr = []
    tr.loss_and_grad(img, first, pol.initial_state(2), actions, upper_grads_ready=lambda: ugr.append(len(log.calls)))
    x0 = tr.last_tape["blocks"][0]["x"]
    assert log.reads(x0, {"col_sums"}) and not log.reads(x0, {"group_sums", "norm_bwd_apply"})
    assert ugr == [len(log.calls)]  # the backward does not enter the CNN: the hook fires at its end
    assert dict(pol.named_parameters())["net.recurrent_layer.blocks.0.pre_r_ln.weight"].grad is not None

    pol, _, _ = make_policy(small_kwargs())
    freeze(pol, "stacks01")
    tr = BCTrainer(pol)
    tr.keep_tape = True
    log = OpLog(monkeypatch, tr)
    tr.loss_and_grad(img, first, pol.initial_state(2), actions, upper_grads_ready=lambda: ugr.append(len(log.calls)))
    stacks = tr.last_tape["stacks"]
    assert stacks[0] is None and stacks[1] is None and stacks[2] is not None
    assert log.names().count("maxpool3s2_bwd") == 1 and "firstconv_bwd" not in log.names()
    assert not log.reads(stacks[2]["x_in"], {"norm_sums", "norm_bwd_apply"})
    assert ugr[-1] < len(log.calls)  # the CNN backward comes after the hook


# ---------------------------------------------------------------------------------------------------------------
# the stored-tape frame limit, and nothing trainable
# ---------------------------------------------------------------------------------------------------------------
def test_frozen_cnn_lifts_the_frame_limit(emu, exact, monkeypatch):
    """cnn_chunk_frames / idm_chunk_frames at 8: a 16-frame call with the CNN frozen runs without recompute_frames (two CNN chunks) and
    gives the oracle's gradient; with stacks 0-1 frozen but stack 2 training it still raises, before anything reaches .grad."""
    pol0, sd, cfg = make_policy(small_kwargs())
    monkeypatch.setattr(type(pol0.net), "cnn_chunk_frames", 8)
    g = torch.Generator().manual_seed(9)
    img, first, actions = batch(g, 2, 8, reset=(1, 5))
    pol = copy.deepcopy(pol0)
    freeze(pol, "stacks01", preset=False)
    with pytest.raises(NotImplementedError):
        BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
    pol.set_autograd(True)
    with pytest.raises(NotImplementedError):
        pol({"img": img}, first, pol.initial_state(2))
    assert all(p.grad is None for p in pol.parameters())

    leaf = oracle_leaf(sd, "cnn")
    (pd_o, _, _), _ = O.agent_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    (-O.logprob(pd_o, actions).mean()).backward()
    grads_o = {k: v.grad for k, v in leaf.items()}
    for autograd in (False, True):
        pol = copy.deepcopy(pol0)
        freeze(pol, "cnn", preset=False)
        if autograd:
            (pd, _, _), _ = pol.set_autograd(True)({"img": img}, first, pol.initial_state(2))
            bc_loss(pol, pd, actions).backward()
        else:
            BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(2), actions)
        assert compare(_grads(pol), grads_o) > 30

    idm0, sd, cfg = make_idm()
    monkeypatch.setattr(type(idm0.net), "idm_chunk_frames", 8)
    img, first, actions = make_batch(g)
    idm = copy.deepcopy(idm0)
    freeze(idm, "stacks01", preset=False)
    with pytest.raises(NotImplementedError):
        IDMTrainer(idm).loss_and_grad(img, first, idm.initial_state(2), actions)
    idm = copy.deepcopy(idm0)
    freeze(idm, "cnn", preset=False)
    IDMTrainer(idm).loss_and_grad(img, first, idm.initial_state(2), actions)
    leaf = oracle_leaf(sd, "cnn")
    (pd_o, _, _), _ = O.idm_policy_forward(leaf, cfg, img, first, O.initial_state(cfg, 2))
    (-O.logprob(pd_o, actions).mean()).backward()
    dense = lambda n: not n.startswith("net.lastlayer.") and not n.endswith((".r_layer.weight", ".r_layer.bias", ".b_nd"))  # noqa: E731
    assert compare({n: v for n, v in _grads(idm).items() if dense(n)}, {k: v.grad for k, v in leaf.items() if dense(k)}) > 10


def test_nothing_trainable_runs_no_backward(emu, monkeypatch):
    """Every parameter frozen: the trainers return the loss and state_out of the all-trainable call and run no backward op."""
    pol0, sd, sd_ref, cfg = test_rl_training.make_pair()
    g = torch.Generator().manual_seed(10)
    img, first, actions = batch(g, 2, 8)
    pd_ref, _ = test_rl_training.ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, 2))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 2))
    rl = test_rl_training.make_rl_batch(g, O.logprob(pd0, actions), 2, 8)
    idm0, _, _ = make_idm()
    img_i, first_i, actions_i = make_batch(g)
    cases = [(BCTrainer, pol0, (img, first, actions), {}),
             (RLTrainer, pol0, (img, first, actions, *rl, pd_ref), dict(vf_coef=0.5, kl_coef=0.1)),
             (IDMTrainer, idm0, (img_i, first_i, actions_i), {})]
    for cls, mod0, args, kw in cases:
        res = []
        for part in (False, True):
            mod = copy.deepcopy(mod0)
            tr = cls(mod)
            if part:
                for p in mod.parameters():
                    p.requires_grad_(False)
                log = OpLog(monkeypatch, tr)
            ugr = []
            loss, st = tr.loss_and_grad(args[0], args[1], mod.initial_state(2), *args[2:], upper_grads_ready=lambda: ugr.append(1), **kw)
            res.append((loss, st))
            assert ugr == [1]
        assert log.names() == [] and all(p.grad is None for p in mod.parameters())
        if cls is BCTrainer:
            assert "softmax_bwd" not in log.names(bwd=False)
        assert torch.equal(res[0][0], res[1][0])
        assert_same_state(res[0][1], res[1][1])
