"""CPU self-check of the float64 forward references (tests/fwd_refs.py): the shape table against hand-written values, and at small shapes
the references (the oracle's unfused layers) against the emulation of the kernels (tests/emu_ops.py) fed the product's own fold tables
(`policy._Prepared`).  The two are written independently, so a wrong reference -- or a wrong fold table -- is caught here without a GPU.
The GPU tests (tests/test_gpu_forward_shapes.py) then hold the kernels to these references at the model's shapes."""
import pytest
import torch

import emu_ops as E
import fwd_refs as Rf
from common import make_policy, small_kwargs
from video_pre_training_b200.policy import _dense_from_zp

BF16, F64 = torch.bfloat16, torch.float64
# the float64 layer vs the emulation with bf16 weights: |err| - 2^-8 |ref| measured at most 3.1e-3 (convs) and 1.9e-3 (linears) of the row max
CONV, LIN = 6e-3, 4e-3


def test_shape_table_follows_the_model():
    s = Rf.forward_shapes("3x")
    assert [(d["H"], d["W"], d["Cin"], d["C"], d["fused_first"]) for d in s["stacks"]] == \
        [(128, 128, 3, 192, True), (64, 64, 192, 384, False), (32, 32, 384, 384, False)]
    assert s["firstconv"] == 192 and s["conv3d"] is None and s["dense"] == (16, 16, 384, 17 * 17 * 384)
    assert (s["h"], s["heads"], s["maxlen"], s["t"], s["causal"], s["qkvr"]) == (3072, 24, 128, 128, True, 9456)
    assert s["head_cols"] == [("camera", 0, 121, 1), ("buttons", 121, 8641, 1)] and (s["ntot"], s["ld_logits"]) == (8762, 8768)
    assert s["linears"] == dict(dense=(256, 110976), linear=(3072, 256), mlp0=(12288, 3072), mlp1=(3072, 12288), proj=(3072, 3072),
                                lastlayer=(3072, 3072))
    assert s["chunk"] == 2048
    s = Rf.forward_shapes("idm")
    assert [(d["H"], d["W"], d["Cin"], d["C"], d["fused_first"]) for d in s["stacks"]] == \
        [(128, 128, 128, 256, False), (64, 64, 256, 512, False), (32, 32, 512, 512, False)]
    assert s["firstconv"] is None and s["conv3d"] == 128 and s["dense"] == (16, 16, 512, 17 * 17 * 512)
    assert (s["h"], s["heads"], s["maxlen"], s["t"], s["causal"], s["qkvr"]) == (4096, 32, 0, 128, False, 3 * 4096)
    assert s["head_cols"] == [("buttons", 0, 2, 20), ("camera", 40, 11, 2)] and (s["ntot"], s["ld_logits"]) == (62, 64)
    assert "lastlayer" not in s["linears"] and s["chunk"] == 512
    assert [d["C"] for d in Rf.forward_shapes("1x")["stacks"]] == [64, 128, 128]


def edge_frames(g, Fn, H, W, C):
    """bf16 ZP frames: randn, post-ReLU-like frames whose mean is several times their spread, one frame whose spread is 1 / 64 of its
    mean (the inputs where a GroupNorm fold cancels most of its bits)"""
    x = torch.randn(Fn, H, W, C, generator=g)
    x[1::2] = x[1::2].relu() + 2.0
    x[-1] = 3.0 + torch.randn(H, W, C, generator=g) * (3.0 / 64)
    return E.to_zp(x.to(BF16))


def close(name, out, ref, floor):
    """|out - ref| <= 2^-8 |ref| + floor * (max |ref| of the row)"""
    d = (out.to(F64) - ref).abs()
    excess = ((d - 2 ** -8 * ref.abs()) / ref.abs().amax(-1, keepdim=True).clamp(min=1e-300)).max().item()
    print(f"{name}: {excess:.2e} (bound {floor:.0e})")
    assert excess <= floor, (name, excess)


@pytest.fixture(scope="module")
def small():
    pol, _, _ = make_policy(small_kwargs(), seed=3)
    sd = {k: v.detach() for k, v in pol.net.state_dict().items()}
    return pol.net, Rf.SD64(sd, "cpu"), pol.net.prepared()


def test_conv_folds_match_the_unfused_layers(small):
    """stack 1's first conv (_fold_conv + the border-class taps), block 0 of stack 1 with the post-pool norm folded in (_fold_conv2,
    norm2_fold, the Ef / affine-residual epilogues) and block 1 (S1 / S2, residual)"""
    net, sd, prep = small
    g = torch.Generator().manual_seed(0)
    st = prep.stacks[1]
    p = "img_process.cnn.stacks.1"
    H, W = net.cfg.img_shape[0] // 2, net.cfg.img_shape[1] // 2
    x = edge_frames(g, 4, H, W, net.cfg.chans[0])
    Wb, S1, S2 = st["first"]
    full, _ = E.conv3x3_zp(x, Wb, H, W, mr=Rf.stats(x, zp=True).float(), S1=S1, S2=S2, relu=1, want_stats=False)
    close("first conv", full[:, :-1, :-1], Rf.conv(x, sd, p + ".firstconv"), CONV)
    H, W = H // 2, W // 2
    C = net.cfg.chans[1]
    y1 = edge_frames(g, 4, H, W, C)
    mrE, Ef, rs, rb = E.norm2_fold(Rf.chan_sums(y1, 2), H * W, st["n_g"], st["n_b"], st["conv0n"][1])
    hmid, _ = E.conv3x3_zp(y1, st["conv0n"][0], H, W, mr=mrE, Ef=Ef, relu=1)
    ref_h, _ = Rf.block(y1, sd, p + ".blocks.0", n=p + ".n")
    close("block 0 conv0 (two-norm fold)", hmid[:, :-1, :-1], ref_h, CONV)
    Wb, S1, S2 = st["convs"][1]
    out, _ = E.conv3x3_zp(hmid, Wb, H, W, mr=Rf.stats(hmid, zp=True).float(), S1=S1, S2=S2, relu=1, residual=y1, res_scale=rs, res_shift=rb)
    x0 = torch.nn.functional.group_norm(Rf.nchw(y1), 1, sd[p + ".n.weight"], sd[p + ".n.bias"], eps=1e-5)
    close("block 0 conv1 (affine residual)", out[:, :-1, :-1], Rf.nhwc(x0) + Rf.conv(hmid, sd, p + ".blocks.0.conv1"), CONV)
    x = edge_frames(g, 4, H, W, C)
    Wb, S1, S2 = st["convs"][2]
    hmid, _ = E.conv3x3_zp(x, Wb, H, W, mr=Rf.stats(x, zp=True).float(), S1=S1, S2=S2, relu=1)
    ref_h, _ = Rf.block(x, sd, p + ".blocks.1")
    close("block 1 conv0", hmid[:, :-1, :-1], ref_h, CONV)


def test_linear_folds_match_the_unfused_layers(small):
    """dense (_dense_to_zp: ZP rows, zero weight columns at the pads), linear / mlp0 / lastlayer (LayerNorm folds), mlp1 and proj (bias,
    residual)"""
    net, sd, prep = small
    cfg = net.cfg
    g = torch.Generator().manual_seed(1)
    Hf, Wf = cfg.final_hw
    xz = edge_frames(g, 6, Hf, Wf, cfg.chans[-1])
    xd = xz.reshape(6, -1)
    mr = Rf.stats(xz, zp=True).float()

    def run(fold, x, N, mr=None, relu=0, residual=None):
        Wb, S1, S2 = fold
        out = torch.empty((x.shape[0], N), dtype=BF16)
        return E.gemm(x, Wb, out, x.shape[0], N, x.shape[1], mr=mr, S1=S1 if mr is not None else None, S2=S2, relu=relu, residual=residual)

    out = run(prep.dense, xd, cfg.cnn_outsize, mr=mr, relu=1)
    close("dense", out, Rf.linear(_dense_from_zp(xd, cfg), sd, "img_process.cnn.dense"), LIN)
    h = cfg.hidsize
    rows = edge_frames(g, 1, 6, 1, h).reshape(-1, h)[:6]
    mr = Rf.stats(rows).float()
    for name, fold, p, n in [("linear", prep.linear, "img_process.linear", h), ("mlp0", prep.layers[0]["mlp0"], "recurrent_layer.blocks.0.mlp0", 4 * h),
                             ("lastlayer", prep.last, "lastlayer", h)]:
        x = rows if name != "linear" else edge_frames(g, 1, 6, 1, 256).reshape(-1, 256)[:6]
        m = mr if name != "linear" else Rf.stats(x).float()
        close(name, run(fold, x, n, mr=m, relu=1), Rf.linear(x, sd, p), LIN)
    a = torch.randn(6, 4 * h, generator=g).to(BF16)
    ref = rows.to(F64) + Rf.linear(a, sd, "recurrent_layer.blocks.0.mlp1", relu=False)
    close("mlp1", run(prep.layers[0]["mlp1"], a, h, residual=rows), ref, LIN)
    a = torch.randn(6, h, generator=g).to(BF16)
    ref = rows.to(F64) + Rf.plain_linear(a, sd, "recurrent_layer.blocks.0.r.orc_block.proj_layer")
    close("proj", run(prep.layers[0]["proj"], a, h, residual=rows), ref, LIN)


def test_plain_nhwc_references_match_the_fp32_mode_forward():
    """precise.forward (the fp32-parity mode) through the emulated ops at the small config, stage by stage: each plain-NHWC reference is fed
    the forward's previous tap, so the stacks (first conv, max-pool, post-pool GroupNorm, blocks), the dense layer on rows flattened H, W, C
    and the linear layer are each held to their float64 layer"""
    from common import emulation
    from video_pre_training_b200 import precise as P

    pol, _, _ = make_policy(small_kwargs(), seed=4)
    net = pol.net
    cfg = net.cfg
    sd = Rf.SD64({k: v.detach() for k, v in net.state_dict().items()}, "cpu")
    B, t = 2, 3
    H, W, _ = cfg.img_shape
    img = torch.randint(0, 256, (B, t, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5))
    net.debug_taps = {}
    try:
        with emulation():
            P.forward(net, img, torch.zeros(B, t, dtype=torch.bool), net.initial_state(B))
        taps = net.debug_taps
    finally:
        net.debug_taps = None

    def near(name, out, ref, bound=1e-4):  # measured 2.6e-5 (the hi / lo splits and fp32 sums of the emulation)
        o, r = out.reshape(out.shape[0], -1).to(F64), ref.reshape(ref.shape[0], -1)
        e = ((o - r).abs().amax(1) / r.pow(2).mean(1).sqrt()).max().item()
        print(f"{name}: max |err| / rms(ref) {e:.2e} (bound {bound:.0e})")
        assert e <= bound, (name, e)

    x = img.reshape(B * t, H, W, 3)
    for i in range(len(cfg.chans)):
        p = f"img_process.cnn.stacks.{i}"
        if i == 0 and not cfg.first_conv_norm:
            pool = Rf.firstconv_pool(x, sd, p)
        else:
            pool = Rf.maxpool_nhwc(Rf.conv_nhwc(x, sd, p + ".firstconv"))
        near(f"stack {i} pool", taps[p + ".pool"], pool)
        x = Rf.group_norm_nhwc(taps[p + ".pool"], sd, p + ".n")
        for j in range(2):
            y = Rf.nhwc(Rf.O.cnn_basic_block(x.to(F64).permute(0, 3, 1, 2), sd, f"{p}.blocks.{j}"))
            near(f"stack {i} block {j}", taps[f"{p}.blocks.{j}"], y)
            x = taps[f"{p}.blocks.{j}"]
    Hf, Wf = cfg.final_hw
    near("dense", taps["img_process.cnn.dense"], Rf.linear(Rf.dense_from_nhwc(x.reshape(B * t, -1), Hf, Wf, cfg.chans[-1]), sd, "img_process.cnn.dense"))
    near("linear", taps["img_process"], Rf.linear(taps["img_process.cnn.dense"], sd, "img_process.linear"))


def test_conv3d_and_firstconv_references_match_emulation():
    g = torch.Generator().manual_seed(2)
    sd = {"c.layer.weight": torch.randn(16, 3, 5, 1, 1, generator=g), "c.layer.bias": torch.randn(16, generator=g) * 0.1,
          "s.firstconv.layer.weight": torch.randn(64, 3, 3, 3, generator=g) * 0.3, "s.firstconv.layer.bias": torch.randn(64, generator=g) * 0.1}
    sd64 = Rf.SD64(sd, "cpu")
    img = torch.randint(0, 256, (2, 7, 4, 4, 3), dtype=torch.uint8, generator=g)
    w3 = (sd["c.layer.weight"].double().reshape(16, 3, 5).permute(0, 2, 1).reshape(16, 15) / 255).float()
    y, _ = E.conv3d_t5(img, w3, sd["c.layer.bias"], 16)
    close("conv3d", y[:, :-1, :-1], Rf.conv3d(img, sd64, "c"), 1e-5)
    img = torch.randint(0, 256, (2, 16, 16, 3), dtype=torch.uint8, generator=g)
    w = (sd["s.firstconv.layer.weight"].double().permute(0, 2, 3, 1).reshape(64, 27) / 255).float()
    y, _ = E.firstconv_pool(img, w, sd["s.firstconv.layer.bias"], 64, zp=True)
    close("firstconv_pool", y[:, :-1, :-1], Rf.firstconv_pool(img, sd64, "s"), 1e-5)
