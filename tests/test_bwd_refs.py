"""CPU self-check of the float64 backward references (tests/bwd_refs.py) against the emulation of the kernels (tests/emu_ops.py) at
small shapes: the two are written independently (autograd / GEMM versus the kernels' own method), so a wrong reference is caught here
without a GPU.  The GPU tests (tests/test_gpu_backward_shapes.py) then hold the kernels to these references at the model's shapes."""
import pytest
import torch

import bwd_refs as Rf
import emu_idm_ops
import emu_ops as E
from video_pre_training_b200.policy import _rot

BF16 = torch.bfloat16


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def zp_rand(g, Fn, H, W, C, relu=False):
    x = torch.randn(Fn, H, W, C, generator=g)
    return E.to_zp((x.relu() if relu else x).to(BF16))


def test_shape_table_follows_the_model():
    s = Rf.backward_shapes("3x")
    assert s["convs"] == [(64, 64, 192, 192), (64, 64, 192, 384), (32, 32, 384, 384), (16, 16, 384, 384)]
    assert s["pools"] == [(64, 64, 384), (32, 32, 384)] and s["gn"] == [(64, 64, 192), (32, 32, 384), (16, 16, 384)]
    assert s["kcat"] == 9456 and s["ld_logits"] == 8768 and s["dense"][3] == 17 * 17 * 384 and s["maxlen"] == 128
    assert s["head_cols"] == [("camera", 0, 121), ("buttons", 121, 8641)]
    assert s["firstconv"] == (128, 128, 192) and (s["h"], s["heads"]) == (3072, 24)
    assert Rf.backward_shapes("1x")["convs"][0] == (64, 64, 64, 64)
    assert [d[0] for d in s["dgrads"]] == ["heads", "heads_value", "lastlayer", "mlp1", "mlp0", "proj", "qkvr", "linear", "dense"]
    assert ("qkvr", 2048, 3072, 9456, True) in s["dgrads"] and ("dense", 2048, 17 * 17 * 384, 256, False) in s["dgrads"]


def test_idm_shape_table_follows_the_model():
    s = Rf.backward_shapes("idm")
    assert (s["N"], s["h"], s["heads"], s["kcat"], s["ld_logits"], s["causal"]) == (512, 4096, 32, 3 * 4096, 64, False)
    assert s["convs"][0] == (128, 128, 128, 256) and s["gn"][0] == (128, 128, 128) and s["pools"][0] == (128, 128, 256)
    assert s["firstconv"] is None and s["dense"] == (16, 16, 512, 147968)
    assert s["head_groups"] == [("buttons", 0, 2, 20), ("camera", 40, 11, 2)]
    assert [d[0] for d in s["dgrads"]] == ["heads", "mlp1", "mlp0", "proj", "qkvr", "linear", "dense"]  # no lastlayer, no value column
    assert ("heads", 512, 4096, 64, False) in s["dgrads"] and ("dense", 512, 147968, 256, False) in s["dgrads"]


def test_conv_references_match_emulation():
    g = torch.Generator().manual_seed(0)
    Fn, H, W, Cin, Cout = 2, 6, 5, 16, 24
    Wt = (torch.randn(Cout, Cin, 3, 3, generator=g) * 0.2).to(BF16)
    dz = zp_rand(g, Fn, H, W, Cout)
    ref, scale = Rf.conv_dgrad(dz, Wt)
    emu, _ = E.conv3x3_zp(dz, _rot(Wt), H, W, relu=0, want_stats=False)   # the rotated layout the dgrad kernel gets
    assert (ref[:, -1] == 0).all() and (ref[:, :, -1] == 0).all()
    assert ((emu.double() - ref).abs() <= 2 ** -8 * ref.abs() + 1e-6 * scale).all()
    u = zp_rand(g, Fn, H, W, Cin)
    ref, scale = Rf.conv_wgrad(dz, u)
    R = Fn * (H + 1) * (W + 1)
    shifts = [(ky - 1) * (W + 1) + (kx - 1) for ky in range(3) for kx in range(3)]
    emu = E.wgrad(dz.reshape(R, Cout), u.reshape(R, Cin), shifts)          # the ZP shift identity
    assert ((emu.double() - ref).abs() <= 1e-6 * scale).all()
    taps, tscale = Rf.conv_wgrad_taps(dz, u)
    assert ((taps - ref).abs() <= 1e-12 * scale).all() and ((tscale - scale).abs() <= 1e-12 * scale).all()


def test_linear_wgrad_reference_matches_emulation():
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn(300, 40, generator=g).to(BF16), torch.randn(300, 24, generator=g).to(BF16)
    ref, scale = Rf.linear_wgrad(a, b)
    assert ((E.wgrad(a, b).double() - ref).abs() <= 1e-6 * scale).all()


@pytest.mark.parametrize("rpg,C,zp", [(8 * 7, 16, (7, 6, 16)), (1, 64, None), (1, 5 * 4 * 8, (4, 3, 8))])
def test_norm_reference_matches_emulation(rpg, C, zp):
    g = torch.Generator().manual_seed(2)
    G = 3
    if zp is None:
        x = (torch.randn(G, C, generator=g) * 0.7 + 0.3).to(BF16)
        du = torch.randn(G, C, generator=g).to(BF16)
    else:
        H, W, Cc = zp
        x = zp_rand(g, G, H, W, Cc).reshape(G * rpg, C)
        du = zp_rand(g, G, H, W, Cc).reshape(G * rpg, C)
    gamma = torch.randn(C, generator=g) * 0.3 + 1
    mr = Rf.norm_stats(x, rpg, zp)
    ref = Rf.norm_bwd(du, x, gamma, rpg, zp)
    count = zp[0] * zp[1] * zp[2] if zp is not None else rpg * C
    ms = E.group_sums(du, x, mr, gamma, rpg, count)
    assert torch.allclose(ms.double(), ref["ms"], rtol=1e-4, atol=1e-6)
    cs = E.col_sums(du, x, mr, rpg)
    assert rel(cs[0], ref["dgamma"]) < 1e-5 and rel(cs[1], ref["dbeta"]) < 1e-6
    dx = E.norm_bwd_apply(du, x, mr, gamma, ref["ms"].float(), rpg, zp=zp)
    assert ((dx.double() - ref["dx"]).abs() <= 2 ** -8 * ref["dx"].abs() + 1e-5 * ref["dx"].abs().max()).all()


@pytest.mark.parametrize("rpg,C,zp", [(8 * 7, 16, (7, 6, 16)), (1, 64, None)])
def test_norm_reference_with_relu_x_and_add_matches_emulation(rpg, C, zp):
    """dx + add, zeroed where the ReLU output x is 0 (the apply pass of a norm whose input is a ReLU output and a residual)"""
    g = torch.Generator().manual_seed(6)
    G = 3
    if zp is None:
        x = (torch.randn(G, C, generator=g) * 0.7 + 0.3).relu().to(BF16)
        du, add = torch.randn(G, C, generator=g).to(BF16), torch.randn(G, C, generator=g).to(BF16)
    else:
        H, W, Cc = zp
        x = zp_rand(g, G, H, W, Cc, relu=True).reshape(G * rpg, C)
        du, add = zp_rand(g, G, H, W, Cc).reshape(G * rpg, C), zp_rand(g, G, H, W, Cc).reshape(G * rpg, C)
    assert (x == 0).float().mean() > 0.2
    gamma = torch.randn(C, generator=g) * 0.3 + 1
    mr = Rf.norm_stats(x, rpg, zp)
    ref = Rf.norm_bwd(du, x, gamma, rpg, zp, add=add, relu_x=True)
    plain = Rf.norm_bwd(du, x, gamma, rpg, zp)
    assert torch.equal(ref["dx"], torch.where(x != 0, plain["dx"] + add.double(), torch.zeros((), dtype=torch.float64)))
    dx = E.norm_bwd_apply(du, x, mr, gamma, ref["ms"].float(), rpg, zp=zp, add=add, relu_x=True)
    assert ((dx.double() - ref["dx"]).abs() <= 2 ** -8 * ref["dx"].abs() + 1e-5 * ref["dx"].abs().max()).all()


@pytest.mark.parametrize("f32", [False, True])
def test_chunked_conv3d_reference_matches_emulation(f32):
    """the frame-chunked float64 conv3d weight gradient against autograd of the whole conv3d: chunks of 3 frames over sequences of 7
    cross the 2-frame time padding at both ends"""
    g = torch.Generator().manual_seed(7)
    B, T, H, W, C = 2, 7, 5, 4, 16
    img = torch.rand(B, T, H, W, 3, generator=g) * 300 - 20 if f32 else torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g)
    dy = E.to_zp(torch.randn(B * T, H, W, C, generator=g).to(BF16))
    ref_w, ref_b = emu_idm_ops.conv3d_t5_bwd(img, dy, C)
    dy[:, -1], dy[:, :, -1] = 3.0, -2.0  # the pad row / column is not part of the conv
    dW, db, sW, sb = Rf.conv3d_t5_wgrad(img, dy, C, chunk=3)
    assert rel(dW, ref_w) < 1e-6 and rel(db, ref_b) < 1e-6
    assert (sW >= dW.abs()).all() and (sb >= db.abs()).all()


def test_maxpool_and_firstconv_references_match_emulation():
    g = torch.Generator().manual_seed(3)
    x = E.to_zp((torch.randn(2, 8, 10, 16, generator=g).relu()).to(BF16))
    dy = zp_rand(g, 2, 4, 5, 16)
    assert torch.equal(Rf.maxpool_bwd(dy, x).to(BF16), E.maxpool3s2_bwd(dy, x))
    img = torch.randint(0, 256, (2, 16, 16, 3), dtype=torch.uint8, generator=g)
    w = torch.randn(64, 27, generator=g) * 0.2 / 255.0
    b = torch.randn(64, generator=g) * 0.1
    dy = zp_rand(g, 2, 8, 8, 64)
    dW, db = Rf.firstconv_bwd(img, w, b, dy)
    dW_e, db_e = E.firstconv_bwd(img, w, b, dy, 64)
    assert rel(dW_e / 255.0, dW) < 1e-5 and rel(db_e, db) < 1e-5   # emulation: w.r.t. the kernel's /255-scaled weights


def test_attention_reference_matches_emulation():
    g = torch.Generator().manual_seed(4)
    B, t, maxlen, heads, nb = 3, 12, 8, 2, 10
    h, T = heads * 128, maxlen + t
    q = (torch.randn(B * t, h, generator=g) * 3).to(BF16)
    kf, vf = torch.randn(B, T, h, generator=g).to(BF16), torch.randn(B, T, h, generator=g).to(BF16)
    R = torch.randn(B * t, heads * nb, generator=g)
    b_nd = torch.randn(nb, maxlen, generator=g) * 0.2
    first = torch.zeros(B, t, dtype=torch.uint8)
    first[1, 0] = 1
    smask = (torch.rand(B, 1, maxlen, generator=g) > 0.3).to(torch.uint8)
    dO = torch.randn(B * t, h, generator=g).to(BF16)
    out = torch.zeros(B * t, 3 * h + heads * nb, dtype=BF16)
    db_e = E.attention_bwd(q, kf, vf, R, b_nd, first, smask, dO, out, B, t, maxlen, heads)
    ref = Rf.attention_bwd(q, kf, vf, R, b_nd, first, smask, dO, B, t, maxlen, heads)
    for name, sl in [("dq", slice(0, h)), ("dk", slice(h, 2 * h)), ("dv", slice(2 * h, 3 * h)), ("dR", slice(3 * h, None))]:
        assert rel(out[:, sl], ref[name]) < 4e-3, name
    assert rel(db_e, ref["db_nd"]) < 1e-5


def test_softmax_reference_matches_emulation():
    g = torch.Generator().manual_seed(5)
    logp = torch.log_softmax(torch.randn(9, 30, generator=g), -1)
    idx = torch.randint(0, 30, (9,), generator=g)
    out = torch.zeros(9, 40, dtype=BF16)
    E.softmax_bwd(logp, idx, 0.5, out, 3)
    ref = Rf.softmax_bwd(logp, idx, 0.5)
    assert torch.equal(out[:, 3:33], ref.to(BF16))
