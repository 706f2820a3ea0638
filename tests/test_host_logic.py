"""CPU: host-side logic of the drop-in policy (schema, init scales, weight re-layout, norm folds, KV bookkeeping) checked
against the oracle by swapping the C-ABI ops for the test-only torch emulation in tests/emu_ops.py."""
import os

import pytest
import torch

import emu_ops
import vpt_b200
import vpt_oracle as O
from common import l2_err, make_policy, rel_err, run_chunks, small_kwargs
from video_pre_training_b200 import ops


@pytest.fixture()
def emulated(monkeypatch):
    for name in dir(emu_ops):
        if not name.startswith("_") and callable(getattr(emu_ops, name)) and hasattr(ops, name):
            monkeypatch.setattr(ops, name, getattr(emu_ops, name))
    yield


def test_state_dict_schema_matches_reference_names():
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "tiny_plain.pt"), weights_only=False)  # reference schema
    pol, _, _ = make_policy(small_kwargs(), pert=False)
    assert list(pol.state_dict().keys()) == [k for k, _, _ in fx["schema"]]
    st = pol.initial_state(3)
    assert len(st) == 2 and st[0][0] is None and st[0][1][0].shape == (3, 8, 256) and st[0][1][0].dtype == torch.float32


def test_load_state_dict_roundtrip():
    a, sd, _ = make_policy(small_kwargs(), seed=1)
    b, _, _ = make_policy(small_kwargs(), seed=2, pert=False)
    missing, unexpected = b.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    assert all(torch.equal(v, b.state_dict()[k]) for k, v in sd.items())


@pytest.mark.parametrize("pert", [False, True])
def test_emulated_forward_matches_oracle(emulated, pert):
    pol, sd, cfg = make_policy(small_kwargs(), pert=pert)
    res = run_chunks(pol, sd, cfg, B=3, chunks=[8, 3, 8, 1], dev="cpu", first_at=(2, 1))
    for r in res:
        for k in r["pd"]:
            assert r["pd"][k].shape == r["pd_o"][k].shape and r["pd"][k].dtype == torch.float32
            assert rel_err(r["pd"][k], r["pd_o"][k]) < 1e-2   # bf16 tolerance of BASELINE.json north_star
        assert (r["v"] - r["v_o"]).abs().max() < 0.1
        for a, b in zip(r["st"], r["st_o"]):
            assert torch.equal(a[0], b[0])
            assert l2_err(a[1][0], b[1][0]) < 5e-2 and l2_err(a[1][1], b[1][1]) < 5e-2


def test_act_api(emulated):
    pol, sd, cfg = make_policy(small_kwargs())
    B = 2
    img = torch.randint(0, 256, (B, 32, 32, 3), dtype=torch.uint8)
    first = torch.zeros(B, dtype=torch.bool)
    torch.manual_seed(3)
    ac, st, res = pol.act({"img": img}, first, pol.initial_state(B), stochastic=True, return_pd=True)
    assert ac["camera"].shape == (B, 1) and ac["buttons"].shape == (B, 1) and ac["buttons"].dtype == torch.int64
    assert res["log_prob"].shape == (B,) and res["vpred"].shape == (B, 1)
    # same uniforms through the oracle's sampler on the returned distribution -> identical actions
    torch.manual_seed(3)
    pd = {k: v.unsqueeze(1) for k, v in res["pd"].items()}
    ac_o = O.sample({"camera": pd["camera"], "buttons": pd["buttons"]})
    assert torch.equal(ac_o["camera"][:, 0], ac["camera"]) and torch.equal(ac_o["buttons"][:, 0], ac["buttons"])
    lp = pol.get_logprob_of_action(pd, ac)
    assert torch.allclose(lp, res["log_prob"])
    pd2, v2, _ = pol.get_output_for_observation({"img": img}, pol.initial_state(B), first)
    assert torch.allclose(pd2["camera"][:, 0], res["pd"]["camera"])


def test_unsupported_configs_are_refused(emulated):
    with pytest.raises(NotImplementedError):
        vpt_b200.MinecraftPolicy(**small_kwargs(recurrence_type="multi_layer_lstm"))
    with pytest.raises(NotImplementedError):
        vpt_b200.MinecraftPolicy(**small_kwargs(hidsize=64))
    pol, _, _ = make_policy(small_kwargs(), pert=False)
    with pytest.raises(AssertionError):
        pol.net._forward_impl(torch.zeros(1, 1, 32, 32, 3, dtype=torch.uint8), torch.zeros(1, 1, dtype=torch.bool), [])


def test_flat_bucket_clip_matches_torch():
    from video_pre_training_b200.parallel import FlatAdamDP

    torch.manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(7, 5)), torch.nn.Parameter(torch.randn(11))]
    ref = [torch.nn.Parameter(p.detach().clone()) for p in params]
    opt = FlatAdamDP(params, lr=1e-3)
    for p, r in zip(params, ref):
        g = torch.randn_like(p) * 3
        p.grad.copy_(g)  # gradients live in the flat bucket
        r.grad = g.clone()
    total_ref = torch.nn.utils.clip_grad_norm_(ref, 5.0)
    total = opt.clip_grad_norm_(5.0)
    assert torch.allclose(total, total_ref) and total > 5.0
    for p, r in zip(params, ref):
        assert torch.allclose(p.grad, r.grad, rtol=1e-6, atol=1e-7)


def test_emulation_mirrors_the_ops_api():
    """The test-only emulation must expose every kernel-launching op of video_pre_training_b200.ops with the same parameter
    names, so that host logic verified against it on CPU is the host logic that drives the kernels."""
    import inspect

    skip = {"require_cuda", "set_default_cluster", "gemm_stat_parts"}
    missing, mismatched = [], []
    for name, fn in vars(ops).items():
        if name.startswith("_") or not inspect.isfunction(fn) or fn.__module__ != ops.__name__ or name in skip:
            continue
        emu = getattr(emu_ops, name, None)
        if emu is None:
            missing.append(name)
            continue
        if list(inspect.signature(fn).parameters) != list(inspect.signature(emu).parameters):
            mismatched.append((name, list(inspect.signature(fn).parameters), list(inspect.signature(emu).parameters)))
    assert not missing, f"ops without an emulation: {missing}"
    assert not mismatched, mismatched


def test_precise_mode_host_logic_matches_oracle(emulated):
    """fp32-parity mode (precise.py): launch order, hi/lo weight splits, explicit norms, KV bookkeeping -- through the emulated ops."""
    pol, sd, cfg = make_policy(small_kwargs())
    pol.set_precision("fp32")
    for o in run_chunks(pol, sd, cfg, 2, [8, 8, 5], "cpu", first_at=(1, 1)):
        for k in o["pd_o"]:
            assert rel_err(o["pd"][k], o["pd_o"][k]) < 1e-4, k
        assert (o["v"] - o["v_o"]).abs().max() < 1e-3
        for (m, (kk, vv)), (m_o, (k_o, v_o)) in zip(o["st"], o["st_o"]):
            assert torch.equal(m, m_o) and torch.allclose(kk, k_o, rtol=1e-3, atol=1e-4) and torch.allclose(vv, v_o, rtol=1e-3, atol=1e-4)
