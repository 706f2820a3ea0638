"""The banded attention kernels for KV memories longer than 128 frames (csrc/attention_long.cuh) on the H100, against float64 references:
the forward, the backward and `vpt_attention_bwd_state` with and without the state gradient / the memory gradient, at maxlen 129 .. 2048,
t 1 .. 128, B 1 .. 16 and 2 or 16 heads (one 2x-width training shape).  Two identical calls give identical bits, the split forward replays
in a CUDA graph, and the shapes the original kernels take (forward while its bias table fits shared memory, backward up to maxlen 128)
still run them."""
import pytest
import torch

import bptt_refs
from test_gpu_bptt import GUARD, PAD, _call, _rel
from video_pre_training_b200 import ops

pytestmark = pytest.mark.gpu

F64 = torch.float64


def fwd_ref(x, B, t, maxlen, heads):
    """float64 attention output [B*t][h] (the forward of tests/bptt_refs.closed_form), computed where the inputs are"""
    Q, Kf, Vf, R, b_nd = x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"]
    dev = Q.device
    h = Q.shape[-1]
    D = h // heads
    T = maxlen + t
    mask, d, okb = bptt_refs._setup(x["first_u8"], x["smask_u8"], B, t, maxlen, dev)
    q = Q.to(F64).reshape(B, t, heads, D).permute(0, 2, 1, 3)
    k = Kf.to(F64).reshape(B, T, heads, D).permute(0, 2, 1, 3)
    v = Vf.to(F64).reshape(B, T, heads, D).permute(0, 2, 1, 3)
    Rh = R.to(F64).reshape(B, t, heads, -1).permute(0, 2, 1, 3)
    Dm = torch.where(okb[None], b_nd.to(F64)[:, d.clamp(0, maxlen - 1)], torch.zeros((), dtype=F64, device=dev))
    S = q @ k.transpose(-1, -2) / D + torch.einsum("bhin,nij->bhij", Rh, Dm)
    P = torch.softmax(S.masked_fill(~mask[:, None], -float("inf")), -1)
    return (P @ v).permute(0, 2, 1, 3).reshape(B * t, h)


def _fwd(x, B, t, maxlen, heads):
    return ops.attention(x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], B, t, maxlen, heads)


FWD_SHAPES = [(1, 1, 1920, 16), (64, 1, 1920, 16), (3, 37, 600, 2), (16, 128, 1920, 16), (1, 128, 2048, 2), (3, 1, 2048, 2), (16, 37, 600, 16)]


@pytest.mark.parametrize("B,t,maxlen,heads", FWD_SHAPES)
def test_forward_matches_float64(B, t, maxlen, heads):
    x = bptt_refs.inputs(B, t, maxlen, heads, seed=B + t + maxlen, dev="cuda", with_dstate=False)
    out = _fwd(x, B, t, maxlen, heads)
    out2 = _fwd(x, B, t, maxlen, heads)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), out2.view(torch.int16)), "not bit-reproducible"
    err = _rel(out, fwd_ref(x, B, t, maxlen, heads))
    print(f"forward B={B} t={t} maxlen={maxlen} heads={heads}: rel-L2 {err:.2e}")
    assert err < 6.8e-3, err


def test_split_forward_replays_in_a_cuda_graph():
    """t = 1 at B = 1 splits each band across a thread-block cluster: capturable, and the replay gives the eager bits"""
    B, t, maxlen, heads = 1, 1, 1920, 16
    x = bptt_refs.inputs(B, t, maxlen, heads, seed=7, dev="cuda", with_dstate=False)
    eager = _fwd(x, B, t, maxlen, heads)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _fwd(x, B, t, maxlen, heads)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _fwd(x, B, t, maxlen, heads)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), eager.view(torch.int16))


BWD_SHAPES = [(3, 1, 129, 16), (2, 128, 129, 2), (3, 37, 600, 2), (2, 1, 1920, 16), (16, 128, 1920, 16), (1, 128, 2048, 2), (4, 37, 2048, 16)]


@pytest.mark.parametrize("B,t,maxlen,heads", BWD_SHAPES)
@pytest.mark.parametrize("with_dstate", [True, False])
def test_backward_matches_float64(B, t, maxlen, heads, with_dstate):
    x = bptt_refs.inputs(B, t, maxlen, heads, seed=B + t + heads + maxlen, dev="cuda", with_dstate=with_dstate)
    h = heads * 128
    nr = 10 * heads
    ld = (3 * h + nr + 7) // 8 * 8 + 16
    ref = bptt_refs.closed_form(x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], x["dO"], B, t, maxlen, heads,
                                dstate=x["dstate"])  # float64 on the GPU
    runs = [_call(x, B, t, maxlen, heads, x["dstate"], True, ld) for _ in range(2)]
    out, db, bufs = runs[0]
    raw = out.view(torch.int16).to(torch.int32) & 0xFFFF
    assert (raw[:, 3 * h + nr:] == GUARD).all(), "guard columns written"
    for buf in bufs:
        assert torch.isnan(buf[:PAD]).all() and torch.isnan(buf[-PAD:]).all(), "dmem guard band written"
        assert torch.isfinite(buf[PAD:-PAD]).all(), "dmem not written in full"
    got = dict(dq=out[:, :h], dk=out[:, h:2 * h], dv=out[:, 2 * h:3 * h], dR=out[:, 3 * h:3 * h + nr], db_nd=db,
               dmem_k=bufs[0][PAD:-PAD].view(B, maxlen, h), dmem_v=bufs[1][PAD:-PAD].view(B, maxlen, h))
    errs = {k: _rel(got[k], ref[k]) for k in got}
    print(f"backward B={B} t={t} maxlen={maxlen} heads={heads} dstate={with_dstate}:", {k: f"{e:.2e}" for k, e in errs.items()})
    for k in ("dq", "dk", "dv", "dR"):
        assert errs[k] < 6.8e-3, (k, errs[k])
    for k in ("db_nd", "dmem_k", "dmem_v"):
        assert errs[k] < 1.4e-6 * 4, (k, errs[k])  # fp32 sums over up to 16x longer bands than tests/test_gpu_bptt.py's
    o2, db2, bufs2 = runs[1]
    assert torch.equal(out.view(torch.int16), o2.view(torch.int16)) and torch.equal(db, db2)
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(bufs, bufs2))
    # without a state gradient, with or without dmem: the columns of vpt_attention_bwd, bit for bit
    args = (x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], x["dO"])
    base = torch.zeros(B * t, ld, dtype=torch.bfloat16, device="cuda")
    db0 = ops.attention_bwd(*args, base, B, t, maxlen, heads)
    for want in (False, True):
        o3 = torch.zeros_like(base)
        db3, dm = ops.attention_bwd_state(*args, o3, B, t, maxlen, heads, dstate=None, want_dmem=want)
        assert torch.equal(o3.view(torch.int16), base.view(torch.int16)) and torch.equal(db3, db0)
        assert (dm is None) == (not want)
    if not with_dstate:
        assert torch.equal(out[:, :3 * h + nr].view(torch.int16), base[:, :3 * h + nr].view(torch.int16))


def _old_forward_fits(maxlen, nbasis=10):
    """vpt_attention's shared-memory budget for its own kernel (csrc/attention.cuh)"""
    smem = (64 + 2 * 64) * 136 * 2 + (64 * maxlen + nbasis * maxlen + 64 * nbasis) * 4 + (maxlen + 15) // 16 * 16 + 16
    return smem <= 227 * 1024


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.key for e in prof.key_averages())


def test_the_original_kernels_keep_their_shapes():
    fit = max(m for m in range(1, 1000) if _old_forward_fits(m))
    assert not _old_forward_fits(fit + 1)
    B, t, heads = 2, 16, 2
    for maxlen, long_fwd in ((fit, False), (fit + 1, True)):
        x = bptt_refs.inputs(B, t, maxlen, heads, seed=1, dev="cuda", with_dstate=False)
        names = _kernels(lambda: _fwd(x, B, t, maxlen, heads))
        assert ("attention_long_kernel" in names) == long_fwd, (maxlen, names)
        assert ("attention_kernel" in names.replace("attention_long_kernel", "")) == (not long_fwd), (maxlen, names)
    for maxlen, long_bwd in ((128, False), (129, True)):
        x = bptt_refs.inputs(B, t, maxlen, heads, seed=2, dev="cuda", with_dstate=True)
        out = torch.zeros(B * t, 3 * heads * 128 + 10 * heads, dtype=torch.bfloat16, device="cuda")
        args = (x["Q"], x["Kf"], x["Vf"], x["R"], x["b_nd"], x["first_u8"], x["smask_u8"], x["dO"])
        names = _kernels(lambda: ops.attention_bwd_state(*args, out, B, t, maxlen, heads, dstate=x["dstate"], want_dmem=True))
        for k in ("attn_bwd_rows", "attn_bwd_keys", "attn_bwd_mem"):
            assert (f"{k}_long_kernel" in names) == long_bwd, (maxlen, k, names)
            assert (f"{k}_kernel" in names) == (not long_bwd), (maxlen, k, names)
        assert "attn_bwd_bnd_kernel" in names
