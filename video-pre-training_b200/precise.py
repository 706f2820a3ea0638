"""fp32-parity precision mode of the forward path (`policy.set_precision("fp32")`; BASELINE north_star "1e-3 rtol fp32").

The reference computes everything in fp32 (lib/xf.py:40 dtype assert, :55-63 fp32 logits).  The production path here multiplies bf16
operands (1e-2 tolerance).  This mode keeps every activation in fp32 and runs each contraction on the SAME wgmma kernel
(`vpt_gemm_bf16`, linear and implicit-GEMM convolution) as three accumulating launches over bf16 hi/lo splits of both operands,

    out = A_hi W_hi^T ;  out += A_lo W_hi^T ;  out = epilogue(out + A_hi W_lo^T)          (fp32 accumulators, fp32 running sum)

which restores ~16 mantissa bits per operand (SURVEY.md section 7.2 measured 7.7e-6 on the logits).  Norms are applied explicitly in
fp32 (csrc/precise.cuh) instead of being folded; attention runs in an fp32 kernel.  It is ~10x slower than the bf16 path and exists
for the parity configurations (BASELINE configs[0], the IDM's near-zero log-probs), not for throughput.

Host code here is launch order and buffer plumbing only; all arithmetic is in libvpt_b200.so.
"""
from collections import OrderedDict

import torch

from . import ops

BF16, F32 = torch.bfloat16, torch.float32


def _split_w(w):
    w = w.detach().float().contiguous()
    hi = w.to(BF16)
    return hi.contiguous(), (w - hi.float()).to(BF16).contiguous()


def _f(t):
    return None if t is None else t.detach().float().contiguous()


class PreparedPrecise:
    """hi/lo bf16 splits of every weight matrix in GEMM layout, norm affines and biases in fp32."""

    def __init__(self, cfg, sd, prefix=""):
        g = lambda k: sd[prefix + k]
        conv_w = lambda k: _split_w(g(k).detach().permute(0, 2, 3, 1).reshape(g(k).shape[0], -1))  # OIHW -> [Cout][tap][Cin]
        p = "img_process.cnn"
        self.conv3d = None
        if cfg.conv3d_out is not None:
            w3 = g("conv3d_layer.layer.weight").detach().double().reshape(cfg.conv3d_out, 3, 5).permute(0, 2, 1).reshape(cfg.conv3d_out, 15) / 255.0
            self.conv3d = (w3.float().contiguous(), _f(g("conv3d_layer.layer.bias")))
        self.stacks = []
        for i, c in enumerate(cfg.chans):
            s = f"{p}.stacks.{i}"
            st = {}
            if i == 0 and not cfg.first_conv_norm:
                w = g(f"{s}.firstconv.layer.weight").detach()
                st["fc_w"] = (w.double().permute(0, 2, 3, 1).reshape(c, 27) / 255.0).float().contiguous()
                st["fc_b"] = _f(g(f"{s}.firstconv.layer.bias"))
            else:
                st["first"] = (conv_w(f"{s}.firstconv.layer.weight"), _f(g(f"{s}.firstconv.norm.weight")), _f(g(f"{s}.firstconv.norm.bias")))
            st["n"] = (_f(g(f"{s}.n.weight")), _f(g(f"{s}.n.bias")))
            st["convs"] = [(conv_w(f"{s}.blocks.{j}.conv{k}.layer.weight"), _f(g(f"{s}.blocks.{j}.conv{k}.norm.weight")),
                            _f(g(f"{s}.blocks.{j}.conv{k}.norm.bias"))) for j in range(2) for k in range(2)]
            self.stacks.append(st)
        C2 = cfg.chans[-1]
        Hf, Wf = cfg.final_hw
        perm = lambda v: v.detach().reshape(*v.shape[:-1], C2, Hf, Wf).movedim(-3, -1).reshape(*v.shape[:-1], -1)  # C,H,W -> H,W,C flatten
        lin = lambda k: (_split_w(g(k + ".layer.weight")), _f(g(k + ".norm.weight")), _f(g(k + ".norm.bias")))
        self.dense = (_split_w(perm(g(f"{p}.dense.layer.weight"))), _f(perm(g(f"{p}.dense.norm.weight"))), _f(perm(g(f"{p}.dense.norm.bias"))))
        self.linear = lin("img_process.linear")
        self.layers = []
        for l in range(cfg.n_layers):
            b = f"recurrent_layer.blocks.{l}"
            o = f"{b}.r.orc_block"
            self.layers.append(dict(
                ln=(_f(g(f"{b}.pre_r_ln.weight")), _f(g(f"{b}.pre_r_ln.bias"))),
                q=(_split_w(g(f"{o}.q_layer.weight")), _f(g(f"{o}.q_layer.bias"))), k=(_split_w(g(f"{o}.k_layer.weight")), None),
                v=(_split_w(g(f"{o}.v_layer.weight")), None), r=(_split_w(g(f"{o}.r_layer.weight")), _f(g(f"{o}.r_layer.bias"))),
                b_nd=_f(g(f"{o}.b_nd")), proj=(_split_w(g(f"{o}.proj_layer.weight")), _f(g(f"{o}.proj_layer.bias"))),
                mlp0=lin(f"{b}.mlp0"), mlp1=(_split_w(g(f"{b}.mlp1.layer.weight")), _f(g(f"{b}.mlp1.layer.bias")))))
        self.last = lin("lastlayer")
        self.fin = (_f(g("final_ln.weight")), _f(g("final_ln.bias")))


def gemm3(xh, xl, W, M, N, K, *, conv=None, bias=None, relu=False, out_scale=1.0, ld=None, acc=None, out=None):
    """fp32 [M][ld >= N] = epilogue(x W^T) with x = xh + xl, W = Wh + Wl (bf16 parts): three wgmma launches (see the module docstring).
    acc / out: fp32 [M][ld] buffers for the running sum and the result (allocated here when not given)."""
    Wh, Wl = W
    ld = ld or N
    if acc is None:
        acc = torch.empty((M, ld), dtype=F32, device=xh.device)
    if out is None:
        out = torch.empty((M, ld), dtype=F32, device=xh.device)
    ops.gemm(xh, Wh, acc, M, N, K, conv=conv, ld_out=ld)
    ops.gemm(xl, Wh, acc, M, N, K, conv=conv, residual=acc, ld_out=ld)        # in place: each element is read, then rewritten, by one thread
    ops.gemm(xh, Wl, out, M, N, K, conv=conv, residual=acc, S2=bias, relu=2 if relu else 0, out_scale=out_scale, ld_out=ld)
    return out


def _norm_gemm(x, rows, C, W, gamma, beta, N, *, conv=None, groups=None, relu=True):
    """[GroupNorm(1) per frame | LayerNorm per row] -> conv3x3 / linear -> [ReLU] (lib/util.py:75-82) in fp32-parity arithmetic."""
    groups = groups or rows
    mr = ops.group_stats_f32(x, groups)
    xh, xl, _ = ops.norm_split_f32(x, mr, gamma, beta, groups=groups)
    K = 9 * C if conv is not None else C
    return gemm3(xh, xl, W, rows, N, K, conv=conv, relu=relu)


def forward(net, img, first, state_in):
    """policy.MinecraftPolicy._forward_impl in the fp32-parity mode -> ((latent hi, latent lo), latent fp32 (B,t,h), state_out)."""
    cfg = net.cfg
    prep = net.prepared_precise()
    B, t = img.shape[:2]
    N = B * t
    H, W = cfg.img_shape[0], cfg.img_shape[1]
    frames = img.reshape(N, H, W, 3).contiguous()  # (uint8 or fp32: policy.frames_f32)
    first_u8 = first.to(device=img.device, dtype=torch.bool).contiguous().view(torch.uint8)
    # ---------------- ImpalaCNN (lib/impala_cnn.py:187-195), NHWC fp32 activations
    x, cin = None, 3
    if prep.conv3d is not None:
        xz, _ = ops.conv3d_t5(img.contiguous(), prep.conv3d[0], prep.conv3d[1], cfg.conv3d_out, out_f32=True)
        x = xz[:, :H, :W, :].contiguous()  # ZP -> plain NHWC (layout plumbing)
        cin = cfg.conv3d_out
        del xz
    for i, c in enumerate(cfg.chans):
        st = prep.stacks[i]
        if "fc_w" in st:
            y1, _ = ops.firstconv_pool(frames, st["fc_w"], st["fc_b"], c, zp=False, out_f32=True)
        else:
            Wf, gam, bet = st["first"]
            full = _norm_gemm(x, N * H * W, cin, Wf, gam, bet, c, conv=(H, W, cin), groups=N)
            y1 = ops.maxpool3s2_f32(full.view(N, H, W, c))
            del full
        H, W = H // 2, W // 2
        net._tap(f"img_process.cnn.stacks.{i}.pool", y1)
        _, _, x = ops.norm_split_f32(y1, ops.group_stats_f32(y1, N), st["n"][0], st["n"][1], groups=N, split=False, want_f32=True)
        del y1
        for j in range(2):
            W0, g0, b0 = st["convs"][2 * j]
            hmid = _norm_gemm(x, N * H * W, c, W0, g0, b0, c, conv=(H, W, c), groups=N)
            W1, g1, b1 = st["convs"][2 * j + 1]
            r = _norm_gemm(hmid, N * H * W, c, W1, g1, b1, c, conv=(H, W, c), groups=N)
            x = ops.add_f32(x, r.view(x.shape))
            net._tap(f"img_process.cnn.stacks.{i}.blocks.{j}", x)
        cin = c
    Kd = H * W * cin
    Wd, gd, bd = prep.dense
    xd = _norm_gemm(x.view(N, Kd), N, Kd, Wd, gd, bd, cfg.cnn_outsize)
    net._tap("img_process.cnn.dense", xd)
    Wl, gl, bl = prep.linear
    h = cfg.hidsize
    x = _norm_gemm(xd, N, cfg.cnn_outsize, Wl, gl, bl, h)
    net._tap("img_process", x)
    # ---------------- transformer (lib/util.py:193-211, lib/xf.py:334-391)
    heads, maxlen = cfg.heads, cfg.maxlen
    causal = cfg.mask_style == "clipped_causal"
    state_out = []
    for l in range(cfg.n_layers):
        L = prep.layers[l]
        state_mask, (mem_k, mem_v) = state_in[l]
        xh, xl, xhat = ops.norm_split_f32(x, ops.group_stats_f32(x, N), L["ln"][0], L["ln"][1], groups=N, want_f32=True)
        q = gemm3(xh, xl, L["q"][0], N, h, h, bias=L["q"][1])
        k = gemm3(xh, xl, L["k"][0], N, h, h)
        v = gemm3(xh, xl, L["v"][0], N, h, h)
        R = gemm3(xh, xl, L["r"][0], N, 10 * heads, h, bias=L["r"][1], ld=(10 * heads + 3) // 4 * 4)[:, :10 * heads].contiguous() if causal else None
        if maxlen > 0:
            if mem_k.shape != (B, maxlen, h):
                raise AssertionError(f"KV memory shape {tuple(mem_k.shape)} != {(B, maxlen, h)}")
            full_k = torch.cat([mem_k.float(), k.view(B, t, h)], 1).contiguous()  # lib/xf.py:378-379 (memory movement only)
            full_v = torch.cat([mem_v.float(), v.view(B, t, h)], 1).contiguous()
        else:
            full_k, full_v = k.view(B, t, h), v.view(B, t, h)
        smask_u8 = state_mask.contiguous().view(torch.uint8) if state_mask is not None else None
        a = ops.attention_f32(q, full_k, full_v, R, L["b_nd"], first_u8, smask_u8, B, t, maxlen, heads, causal=causal)
        T = maxlen + t
        new_k = full_k[:, T - maxlen:].contiguous()  # lib/xf.py:380-381
        new_v = full_v[:, T - maxlen:].contiguous()
        new_mask = ops.state_mask_update(smask_u8, first_u8, t, maxlen) if causal else state_mask
        state_out.append((new_mask, (new_k, new_v)))
        ah, al, _ = ops.norm_split_f32(a)
        y = ops.add_f32(xhat, gemm3(ah, al, L["proj"][0], N, h, h, bias=L["proj"][1]))
        net._tap(f"recurrent_layer.blocks.{l}.attn", y)
        W0, g0, b0 = L["mlp0"]
        hmid = _norm_gemm(y, N, h, W0, g0, b0, h * cfg.pointwise_ratio)
        hh, hl, _ = ops.norm_split_f32(hmid)
        last = l == cfg.n_layers - 1
        x = ops.add_f32(y, gemm3(hh, hl, L["mlp1"][0], N, h, h * cfg.pointwise_ratio, bias=L["mlp1"][1]), relu=last)  # F.relu of lib/policy.py:211
        if not last:
            net._tap(f"recurrent_layer.blocks.{l}", x)
    if net.use_lastlayer:
        Wt, gt, bt = prep.last
        x = _norm_gemm(x, N, h, Wt, gt, bt, h)
    lh, ll, lat = ops.norm_split_f32(x, ops.group_stats_f32(x, N), prep.fin[0], prep.fin[1], groups=N, want_f32=True)
    return (lh, ll), lat.view(B, t, h), state_out


def heads(pol, lat, B, t, mask=None):
    """policy._PolicyBase._heads in the fp32-parity mode (lib/action_head.py:163-174, lib/scaled_mse_head.py:34-35)."""
    lh, ll = lat
    N, h = lh.shape
    hp = pol._heads_prepared_precise()
    ntot = hp["ntot"]
    ld = (ntot + 7) // 8 * 8
    raw = gemm3(lh, ll, hp["pi"][0], N, ntot, h, bias=hp["pi"][1], out_scale=1.0 / pol.temperature, ld=ld)
    pd = OrderedDict()
    for name, (shape, n) in pol.head_specs.items():
        c0, width = hp["cols"][name]
        cnt = width // n
        if mask is not None and mask.get(name) is not None:
            view = raw[:, c0:c0 + width].view(B, t, *shape, n)
            view.masked_fill_(~mask[name].to(device=raw.device, dtype=torch.bool).expand_as(view), -100.0)
        lp = ops.log_softmax(raw, c0, n) if cnt == 1 else torch.cat([ops.log_softmax(raw, c0 + i * n, n) for i in range(cnt)], dim=1)
        pd[name] = lp.view(B, t, *shape, n)
    if not pol.has_value_head:
        return pd, None
    vpred = gemm3(lh, ll, hp["v"][0], N, 1, h, bias=hp["v"][1], ld=4)[:, :1].contiguous()
    return pd, vpred.view(B, t, 1)
