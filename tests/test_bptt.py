"""Truncated backpropagation through time across calls (`set_autograd(True, state_grad=True)`) on the CPU: `loss.backward()` through the
test-only torch emulation of the ops (tests/emu_ops.py and friends, tests/emu_bptt_ops.py for the attention backward through the KV memory)
against autograd through the oracle with the state NOT detached, at the SMALL config (maxlen 8).  tests/test_gpu_bptt.py repeats it through
the CUDA kernels."""
import contextlib
import inspect

import pytest
import torch

import bptt_refs
import emu_bptt_ops
import vpt_oracle as O
from common import make_policy, small_kwargs
from test_autograd import _with_grad, batch, bc_loss, compare, emulated, exact, leaf_of  # noqa: F401  (fixtures)
from test_idm_training import make_batch, make_idm
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops, ops_bptt


@pytest.fixture()
def bptt(emulated, monkeypatch):  # noqa: F811
    monkeypatch.setattr(ops, "attention_bwd_state", _with_grad(emu_bptt_ops.attention_bwd_state))
    yield


def _leaf_state(st):
    """A copy of the state whose K / V are leaves that require grad."""
    return [(m, (k.detach().clone().requires_grad_(True), v.detach().clone().requires_grad_(True))) for m, (k, v) in st]


def _param_grads(pol):
    return {n: p.grad for n, p in pol.named_parameters()}


def _state_err(st, st_o):
    worst = 0.0
    for (_, (k, v)), (_, (k_o, v_o)) in zip(st, st_o):
        for a, b in ((k, k_o), (v, v_o)):
            assert (a.grad is None) == (b.grad is None)
            if b.grad is not None and b.grad.any():
                worst = max(worst, ((a.grad - b.grad).norm() / b.grad.norm()).item())
    return worst


def test_two_chunks_bc_on_both_is_the_exact_gradient(bptt, exact):
    """Two chunks of t = 8 (B = 2, an episode reset at the start of row 1's second chunk), the BC loss on both, ONE backward with the state
    carried attached: the oracle's autograd through the memory, value_head.* None."""
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(0)
    B, T = 2, 8
    leaf = leaf_of(sd)
    st, st_o = pol.initial_state(B), O.initial_state(cfg, B)
    loss = loss_o = 0.0
    for c in range(2):
        img, first, actions = batch(g, B, T, reset=(1, 0) if c == 1 else None)
        (pd, _, _), st = pol({"img": img}, first, st)
        assert all(k.requires_grad and v.requires_grad for _, (k, v) in st)
        loss = loss + bc_loss(pol, pd, actions)
        (pd_o, _, _), st_o = O.agent_policy_forward(leaf, cfg, img, first, st_o)
        loss_o = loss_o - O.logprob(pd_o, actions).mean()
    loss.backward()
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    grads = _param_grads(pol)
    assert grads["value_head.linear.weight"] is None
    assert compare(grads, {k: v.grad for k, v in leaf.items()}) > 40


def test_uneven_chunks_loss_on_last_reaches_the_state(bptt, exact):
    """Chunks of t = 3, 3, 5 (t < maxlen: state_out rows that are memory rows pass straight through) from a leaf state filled by a no_grad
    warm-up chunk, the loss on the last chunk only: the parameter gradients AND the gradient wrt the leaf state match the oracle's."""
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(1)
    B = 2
    img, first, _ = batch(g, B, 8)
    with torch.no_grad():
        _, st0 = pol({"img": img}, first, pol.initial_state(B))
    st, st_o = _leaf_state(st0), _leaf_state(st0)
    s, s_o = st, st_o
    leaf = leaf_of(sd)
    for c, t in enumerate((3, 3, 5)):
        img, first, actions = batch(g, B, t, reset=(0, 0) if c == 1 else None)
        (pd, _, _), s = pol({"img": img}, first, s)
        (pd_o, _, _), s_o = O.agent_policy_forward(leaf, cfg, img, first, s_o)
    loss = bc_loss(pol, pd, actions)
    loss_o = -O.logprob(pd_o, actions).mean()
    loss.backward()
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    assert compare(_param_grads(pol), {k: v.grad for k, v in leaf.items()}) > 40
    assert all(k.grad is not None and k.grad.any() and v.grad.any() for _, (k, v) in st)
    assert _state_err(st, st_o) < 1e-3


def test_reference_loop_shape_one_backward(bptt, exact):
    """The reference BC loop's shape (B = 1, T = 1) over six calls with the state kept attached and ONE backward of the summed loss."""
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(2)
    leaf = leaf_of(sd)
    st, st_o = pol.initial_state(1), O.initial_state(cfg, 1)
    loss = loss_o = 0.0
    for _ in range(6):
        img, first, actions = batch(g, 1, 1)
        (pd, _, _), st = pol({"img": img}, first, st)
        (pd_o, _, _), st_o = O.agent_policy_forward(leaf, cfg, img, first, st_o)
        loss = loss + bc_loss(pol, pd, actions) / 6
        loss_o = loss_o - O.logprob(pd_o, actions).mean() / 6
    loss.backward()
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 1e-4 * abs(loss_o.item())
    assert compare(_param_grads(pol), {k: v.grad for k, v in leaf.items()}) > 40


def window_vs_forced(pol, sd, cfg, chunks, loss_on, ctx=contextlib.nullcontext, st=None):
    """`chunks` [(img, first, actions)] as one window with the state attached (from `st`, detached, or the initial state) and ONE backward
    of the BC loss on the chunks in `loss_on`, against autograd through the BPTT forced replica of the calls' own tapes (run inside `ctx()`)
    -> (loss, replica loss, {param: rel-L2})."""
    from forced_replica_bptt import forced_window
    from video_pre_training_b200.policy import _autograd_runner

    runner = _autograd_runner(pol)
    runner.keep_tape = True
    st = pol.initial_state(chunks[0][0].shape[0]) if st is None else st
    tapes, loss = [], 0.0
    for c, (img, first, actions) in enumerate(chunks):
        (pd, _, _), st = pol({"img": img}, first, st)
        tapes.append(runner.last_tape)
        if c in loss_on:
            loss = loss + bc_loss(pol, pd, actions)
    loss.backward()
    runner.keep_tape, runner.last_tape = False, None
    leaf = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.startswith("value_head.normalizer.")) for k, v in sd.items()}
    with ctx():
        pds = forced_window(leaf, cfg, tapes, [(img, first) for img, first, _ in chunks])
        loss_f = sum(-O.logprob(pds[c], chunks[c][2]).mean() for c in loss_on)
        loss_f.backward()
    worst = {}
    for n, p in pol.named_parameters():
        assert (p.grad is None) == (leaf[n].grad is None), n
        if p.grad is not None and leaf[n].grad.any():
            worst[n] = ((p.grad - leaf[n].grad).norm() / leaf[n].grad.norm()).item()
    return loss.item(), loss_f.item(), worst


def test_bf16_emulation_two_chunks_matches_forced_replica(bptt):
    """Every bf16 rounding point of the emulation active: two chunks with the BC loss on both against the BPTT forced replica (autograd at
    the emulated forward's operating point, the memory rows being the first chunk's forced K / V)."""
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(3)
    chunks = [batch(g, 2, 8, reset=(1, 0) if c == 1 else None) for c in range(2)]
    loss, loss_f, worst = window_vs_forced(pol, sd, cfg, chunks, (0, 1))
    assert abs(loss - loss_f) < 1e-3 * abs(loss_f)
    print("bf16 emulation vs BPTT forced replica, worst", sorted(worst.items(), key=lambda kv: -kv[1])[:4])
    assert max(worst.values()) < 3e-2, sorted(worst.items(), key=lambda kv: -kv[1])[:4]


def test_flag_with_detached_state_is_bit_identical(bptt):
    """state_grad on, the caller detaching the state after every chunk and calling backward per chunk: bit for bit the flag-off gradients."""
    pol, _, _ = make_policy(small_kwargs())
    g0 = torch.Generator().manual_seed(4)
    chunks = [batch(g0, 2, 8, reset=(0, 0) if c == 1 else None) for c in range(2)]
    res = []
    for sg in (False, True):
        pol.zero_grad(set_to_none=True)
        pol.set_autograd(True, state_grad=sg)
        st = pol.initial_state(2)
        for img, first, actions in chunks:
            (pd, _, _), st = pol({"img": img}, first, st)
            assert all(k.requires_grad == sg for _, (k, v) in st)
            st = [(m, (k.detach(), v.detach())) for m, (k, v) in st]
            bc_loss(pol, pd, actions).backward()
        res.append({n: None if p.grad is None else p.grad.clone() for n, p in pol.named_parameters()})
    for n in res[0]:
        assert (res[0][n] is None) == (res[1][n] is None), n
        assert res[0][n] is None or torch.equal(res[0][n], res[1][n]), n


def test_default_refuses_and_window_backward_raises(bptt):
    pol, _, _ = make_policy(small_kwargs())
    g = torch.Generator().manual_seed(5)
    img, first, actions = batch(g, 1, 8)
    pol.set_autograd(True)
    with pytest.raises(ValueError, match="state_grad"):  # the default still refuses a state_in that requires grad
        pol({"img": img}, first, _leaf_state(pol.initial_state(1)))
    pol.set_autograd(True, state_grad=True)
    (pd, _, _), st = pol({"img": img}, first, pol.initial_state(1))
    bc_loss(pol, pd, actions).backward()  # frees chunk 1's tape
    (pd, _, _), _ = pol({"img": img}, first, st)
    with pytest.raises(RuntimeError, match="detach the state or call backward once per window"):
        bc_loss(pol, pd, actions).backward()
    pol.set_autograd(False)
    assert not pol._state_grad and not pol.net._state_grad


def test_bare_network_loss_on_second_chunk(bptt, exact):
    """MinecraftPolicy on its own: a loss on the second chunk's latent only reaches the first chunk through the memory."""
    pol, sd, cfg = make_policy(small_kwargs())
    net = pol.net.set_autograd(True, state_grad=True)
    g = torch.Generator().manual_seed(6)
    leaf = leaf_of(sd)
    st, st_o = net.initial_state(2), O.initial_state(cfg, 2)
    for c in range(2):
        img, first, _ = batch(g, 2, 8)
        (lat, _), st = net({"img": img}, st, {"first": first})
        lat_o, st_o = O.minecraft_policy_forward(leaf, cfg, img, first, st_o)
    w = torch.randn(2, 8, cfg.hidsize, generator=g)
    (lat * w).sum().backward()
    (lat_o * w).sum().backward()
    grads_o = {k[4:]: v.grad for k, v in leaf.items() if k.startswith("net.")}
    assert compare({n: p.grad for n, p in net.named_parameters()}, grads_o) > 30


def test_idm_is_unaffected(bptt):
    """The IDM has no memory (maxlen 0): state_grad changes nothing, bit for bit, and the state stays detached."""
    res = []
    for sg in (False, True):
        idm, _, _ = make_idm()
        idm.set_autograd(True, state_grad=sg)
        g = torch.Generator().manual_seed(0)
        img, first, actions = make_batch(g)
        (pd, _, _), st = idm({"img": img}, first, idm.initial_state(2))
        assert all(not k.requires_grad and not v.requires_grad for _, (k, v) in st)
        (-idm.logprob(actions, pd).mean()).backward()
        res.append({n: None if p.grad is None else p.grad.clone() for n, p in idm.named_parameters()})
        with pytest.raises(ValueError):
            idm({"img": img}, first, _leaf_state(idm.initial_state(2)))
    for n in res[0]:
        assert (res[0][n] is None) == (res[1][n] is None), n
        assert res[0][n] is None or torch.equal(res[0][n], res[1][n]), n


@pytest.mark.parametrize("B,t,maxlen,heads", [(2, 8, 8, 2), (3, 3, 8, 1), (2, 1, 8, 2), (2, 20, 16, 1)])
@pytest.mark.parametrize("with_dstate", [False, True])
def test_kernel_reference_matches_autograd(B, t, maxlen, heads, with_dstate):
    """The float64 closed form the GPU test checks the kernel against equals torch autograd with the memory rows as leaves."""
    x = bptt_refs.inputs(B, t, maxlen, heads, seed=B * 100 + t, with_dstate=with_dstate)
    args = (x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], x["dO"], B, t, maxlen, heads)
    a = bptt_refs.closed_form(*args, dstate=x["dstate"])
    b = bptt_refs.by_autograd(*args, dstate=x["dstate"])
    for key in a:
        scale = b[key].abs().max().item()
        assert (a[key] - b[key]).abs().max().item() <= 1e-10 * max(scale, 1.0), key
    assert b["dmem_k"].abs().max() > 0 and b["dmem_v"].abs().max() > 0
    # first-reset rows see no memory: their memory gradient is the state_out pass-through alone
    fr = x["first_u8"][:, 0] != 0
    pt = torch.zeros(B, maxlen, 128 * heads, dtype=torch.float64)
    if with_dstate and t < maxlen:
        pt[:, t:] = x["dstate"][0][:, :maxlen - t].double()
    assert torch.equal(a["dmem_k"][fr], pt[fr])


def test_emulation_and_abi_mirror_the_op():
    assert ops.attention_bwd_state is ops_bptt.attention_bwd_state
    assert list(inspect.signature(ops_bptt.attention_bwd_state).parameters) == \
        list(inspect.signature(emu_bptt_ops.attention_bwd_state).parameters)
    assert "vpt_attention_bwd_state" in nat.SIGNATURES
    assert len(nat.SIGNATURES["vpt_attention_bwd_state"][1]) == len(nat.SIGNATURES["vpt_attention_bwd"][1]) + 4
