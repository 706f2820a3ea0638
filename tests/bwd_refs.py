"""TEST-ONLY float64 references of the BC backward operations, and the backward call shapes of the released models.

Each reference takes the same bf16 / fp32 inputs the kernel gets and restates the *mathematical* operation -- autograd of the
forward op or a plain GEMM -- in float64 plain torch (any device).  They do not copy the kernels' method the way tests/emu_ops.py
does: the conv weight gradient is `conv2d_weight` on the ZP interiors (not the ZP shift identity of `wgrad`), the dgrad conv
uses the original [Cout, Cin, 3, 3] weight (not the rotated layout the kernel runs on), so an error in one of those assumptions
shows up here.  `backward_shapes` derives every shape from the model config, so the tests follow the model when it changes."""
import torch
import torch.nn.functional as F

import vpt_b200
import vpt_oracle as O
from video_pre_training_b200.policy import NetConfig

F64 = torch.float64
NBASIS = 10


# ---------------------------------------------------------------------------------------------------------------------
# shapes
# ---------------------------------------------------------------------------------------------------------------------
def backward_shapes(width, B=None, T=128):
    """The call shapes the backward (training.py) reaches for the released model `width`: `policy_kwargs(width)` (1x / 2x / 3x, the BC
    and RL steps, B = 16) or `idm_net_kwargs()` ("idm", B = 4: the 512 frames of `idm_chunk_frames`), at B x T frames / tokens.

    head_cols lists (name, first column, columns) of the logits gradient, head_groups (name, first column, classes, sub-actions) (the
    IDM's factored heads: 20 x 2 and 2 x 11).  dgrads lists the input-gradient GEMMs `_gemm` runs, (name, M, N, K, residual):
    out [M][N] = dz [M][K] @ W_t[N][K]^T; "heads_value" is the RL step's heads GEMM with the value head's column."""
    idm = width == "idm"
    cfg = NetConfig(**(vpt_b200.idm_net_kwargs() if idm else vpt_b200.policy_kwargs(width)))
    B = B or (4 if idm else 16)
    H0, W0, _ = cfg.img_shape
    c = cfg.chans
    h, heads = cfg.hidsize, cfg.heads
    causal = cfg.mask_style == "clipped_causal"
    Hf, Wf = cfg.final_hw
    kd = (Hf + 1) * (Wf + 1) * c[-1]                 # dense input row in ZP (h, w, c) order
    kcat = (3 * h + NBASIS * heads + 7) // 8 * 8 if causal else 3 * h  # q | k | v [| R] gradient buffer (training.py)
    space = vpt_b200.idm_action_space() if idm else vpt_b200.minecraft_action_space()
    cols, groups, c0 = [], [], 0
    for name, sp in space.items():
        n, cnt = sp.eltype.n, 1
        for d in sp.shape:
            cnt *= d
        cols.append((name, c0, n * cnt))
        groups.append((name, c0, n, cnt))
        c0 += n * cnt
    ld_logits = (c0 + 7) // 8 * 8
    # 3x3 convs of the CNN backward, (H, W, Cin, Cout) at their frame size: stack i > 0 (and the IDM's stack 0) opens with a normalised
    # conv at the stack's input size, followed by the max-pool
    convs, norms, pools = [], [], []
    Hs, Ws, cin = H0, W0, cfg.conv3d_out
    for i, C in enumerate(c):
        if i > 0 or cfg.first_conv_norm:
            convs.append((Hs, Ws, cin, C))
            if i == 0:
                norms.append((Hs, Ws, cin))              # the GroupNorm(1) of the conv3d output
            pools.append((Hs, Ws, C))                    # max-pool backward input (pre-pool size)
        Hs, Ws, cin = Hs // 2, Ws // 2, C
        convs.append((Hs, Ws, C, C))
        norms.append((Hs, Ws, C))                        # GroupNorm(1) ZP frames of this stack
    assert (Hs, Ws) == (Hf, Wf)
    uniq = lambda v: list(dict.fromkeys(v))
    N, f = B * T, h * cfg.pointwise_ratio
    dgrads = [("heads", N, h, ld_logits, False)]
    if not idm:
        dgrads += [("heads_value", N, h, (c0 + 1 + 7) // 8 * 8, False), ("lastlayer", N, h, h, False)]
    dgrads += [("mlp1", N, f, h, False), ("mlp0", N, h, f, False), ("proj", N, h, h, False), ("qkvr", N, h, kcat, True),
               ("linear", N, cfg.cnn_outsize, h, False), ("dense", N, kd, cfg.cnn_outsize, False)]
    return dict(
        cfg=cfg, B=B, T=T, N=N, h=h, heads=heads, maxlen=cfg.maxlen, causal=causal, kcat=kcat, ld_logits=ld_logits, head_cols=cols,
        head_groups=groups, convs=uniq(convs), gn=uniq(norms), pools=uniq(pools), firstconv=None if cfg.first_conv_norm else (H0, W0, c[0]),
        ln=uniq([h, cfg.cnn_outsize]), dense=(Hf, Wf, c[-1], kd), dgrads=dgrads,
        linears=uniq([(ld_logits, h), (kcat, h), (h, f), (f, h), (h, h), (h, cfg.cnn_outsize), (cfg.cnn_outsize, kd)]),
    )


# ---------------------------------------------------------------------------------------------------------------------
# ZP helpers (ZP = [F, H+1, W+1, C] with a zero last row / column)
# ---------------------------------------------------------------------------------------------------------------------
def nchw(zp):
    return zp[:, :-1, :-1, :].to(F64).permute(0, 3, 1, 2)


def to_zp(x_nchw):
    return F.pad(x_nchw.permute(0, 2, 3, 1), (0, 0, 0, 1, 0, 1))


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def conv_dgrad(dz, W):
    """d/dx of conv2d(x, W, padding=1): dz ZP [F,H+1,W+1,Cout], W [Cout, Cin, 3, 3] -> (ZP float64 [F,H+1,W+1,Cin], same op on
    |dz|, |W| = the scale of each output's sum)."""
    Fn, H, Wd = dz.shape[0], dz.shape[1] - 1, dz.shape[2] - 1
    shape = (Fn, W.shape[1], H, Wd)
    g = torch.nn.grad.conv2d_input(shape, W.to(F64), nchw(dz), padding=1)
    s = torch.nn.grad.conv2d_input(shape, W.to(F64).abs(), nchw(dz).abs(), padding=1)
    return to_zp(g), to_zp(s)


def conv_wgrad(dz, u):
    """d/dW of conv2d(u, W, padding=1) on the ZP interiors, as [Cout][tap][Cin] (tap = ky*3 + kx), and the same op on |dz|, |u|."""
    Cout, Cin = dz.shape[3], u.shape[3]
    perm = lambda w: w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin)
    g = torch.nn.grad.conv2d_weight(nchw(u), (Cout, Cin, 3, 3), nchw(dz), padding=1)
    s = torch.nn.grad.conv2d_weight(nchw(u).abs(), (Cout, Cin, 3, 3), nchw(dz).abs(), padding=1)
    return perm(g), perm(s)


def conv_wgrad_taps(dz, u):
    """conv_wgrad as nine float64 GEMMs over the zero-padded interiors (dW[:, tap] = dz^T u shifted by the tap), for frame counts where
    a float64 convolution is slow; [Cout][tap][Cin] and the same over |dz|, |u|."""
    H, W = dz.shape[1] - 1, dz.shape[2] - 1
    Cout, Cin = dz.shape[3], u.shape[3]
    g = dz[:, :H, :W].to(F64).reshape(-1, Cout)
    up = F.pad(u[:, :H, :W].to(F64), (0, 0, 1, 1, 1, 1))
    taps = [up[:, ky:ky + H, kx:kx + W].reshape(-1, Cin) for ky in range(3) for kx in range(3)]
    return torch.cat([g.T @ x for x in taps], 1), torch.cat([g.abs().T @ x.abs() for x in taps], 1)


def linear_wgrad(a, b):
    """a^T b over the rows, and |a|^T |b|."""
    a, b = a.to(F64), b.to(F64)
    return a.T @ b, a.abs().T @ b.abs()


def norm_stats(x, rows_per_group, zp=None):
    """(mean, rstd) per group of the real (non-pad) elements, float64 -> fp32 [G, 2] (what the forward hands the backward)."""
    xi = _real(x.to(F64), rows_per_group, zp)
    mean = xi.mean(1)
    var = xi.var(1, unbiased=False)
    return torch.stack([mean, 1 / torch.sqrt(var + 1e-5)], 1).float()


def _real(v, rows_per_group, zp):
    """[rows][C] -> [G][real elements of the group] (ZP pads dropped)"""
    G = v.shape[0] // rows_per_group
    if zp is None:
        return v.reshape(G, -1)
    H, W, Cc = zp
    return v.reshape(G, H + 1, W + 1, Cc)[:, :H, :W].reshape(G, -1)


def norm_bwd(du, x, gamma, rows_per_group, zp=None, add=None, relu_x=False):
    """Autograd of GroupNorm(1) over a ZP frame (rows_per_group > 1) or LayerNorm over a row (rows_per_group == 1; with zp the row
    is a ZP image whose pads are not part of the norm) in float64.  gamma: fp32 [C].  add: a gradient that reaches x by another path
    (a residual), added to dx; relu_x: x is the output of a ReLU, whose backward then zeroes the total where x == 0.
    Returns dict(dx [rows][C] (zero at pads), dgamma [C], dbeta [C], ms [G][2] = (mean gamma*du, mean gamma*du*n))."""
    r = _norm_bwd(du, x, gamma, rows_per_group, zp)
    if add is not None:
        r["dx"] = r["dx"] + add.to(F64).reshape(r["dx"].shape)
    if relu_x:
        r["dx"] = torch.where(x.reshape(r["dx"].shape) != 0, r["dx"], torch.zeros((), dtype=F64, device=x.device))
    return r


def _norm_bwd(du, x, gamma, rows_per_group, zp):
    rows, C = x.shape
    G = rows // rows_per_group
    dev = x.device
    if rows_per_group > 1:  # GroupNorm(1): one frame per group, per-channel affine
        H, W, Cc = zp
        xi = x.to(F64).reshape(G, H + 1, W + 1, Cc)[:, :H, :W].permute(0, 3, 1, 2).clone().requires_grad_(True)
        gi = du.to(F64).reshape(G, H + 1, W + 1, Cc)[:, :H, :W].permute(0, 3, 1, 2)
        g = gamma.to(F64).clone().requires_grad_(True)
        b = torch.zeros(C, dtype=F64, device=dev, requires_grad=True)
        y = F.group_norm(xi, 1, g, b, eps=1e-5)
        dxi, dg, db = torch.autograd.grad(y, (xi, g, b), gi)
        n = F.group_norm(xi.detach(), 1, eps=1e-5)
        gdu = gi * gamma.to(F64)[None, :, None, None]
        dx = to_zp(dxi).reshape(rows, C)
    else:                   # LayerNorm over the real elements of each row, per-element affine
        xi = _real(x.to(F64), 1, zp).clone().requires_grad_(True)
        gi = _real(du.to(F64), 1, zp)
        g = _real(gamma.to(F64)[None], 1, zp)[0].clone().requires_grad_(True)
        b = torch.zeros_like(g, requires_grad=True)
        y = F.layer_norm(xi, (xi.shape[1],), g, b, eps=1e-5)
        dxi, dgi, dbi = torch.autograd.grad(y, (xi, g, b), gi)
        n = F.layer_norm(xi.detach(), (xi.shape[1],), eps=1e-5)
        gdu = gi * g.detach()
        if zp is None:
            dx, dg, db = dxi, dgi, dbi
        else:
            H, W, Cc = zp
            put = lambda v: F.pad(v.reshape(-1, H, W, Cc), (0, 0, 0, 1, 0, 1)).reshape(v.shape[0], -1)
            dx, dg, db = put(dxi), put(dgi[None])[0], put(dbi[None])[0]
    count = n[0].numel()
    ms = torch.stack([gdu.reshape(G, -1).sum(1) / count, (gdu * n).reshape(G, -1).sum(1) / count], 1)
    return dict(dx=dx, dgamma=dg, dbeta=db, ms=ms)


def maxpool_bwd(dy, x):
    """Autograd of max_pool2d(ReLU(x), 3, 2, 1) on ZP tensors (x: the post-ReLU pool input) -> ZP float64 dx."""
    xi = nchw(x).requires_grad_(True)
    (g,) = torch.autograd.grad(F.max_pool2d(F.relu(xi), 3, 2, 1), xi, nchw(dy))
    return to_zp(g)


def firstconv_bwd(img, w, bias, dy):
    """Autograd of u8/255 -> conv3x3(W, b) -> ReLU -> max_pool2d(3, 2, 1).  w: the kernel's fp32 [C0][27] = W[c0][ky][kx][c] / 255.
    Returns (dW [C0][27] in (ky, kx, c) order, db [C0]) with respect to the model's W and b."""
    C0 = w.shape[0]
    x = img.to(F64).permute(0, 3, 1, 2) / 255.0
    W = (w.to(F64) * 255.0).reshape(C0, 3, 3, 3).permute(0, 3, 1, 2).clone().requires_grad_(True)  # OIHW
    b = bias.to(F64).clone().requires_grad_(True)
    y = F.max_pool2d(F.relu(F.conv2d(x, W, b, padding=1)), 3, 2, 1)
    dW, db = torch.autograd.grad(y, (W, b), nchw(dy))
    return dW.permute(0, 2, 3, 1).reshape(C0, 27), db


def attention_bwd(Q, Kf, Vf, R, b_nd, first_u8, smask_u8, dO, B, t, maxlen, heads):
    """Autograd of the clipped-causal attention with relative-position logits (the formulas of tests/forced_replica.py, from the
    oracle) in float64.  The memory rows of K / V are constants.  Returns dict(dq, dk, dv [B*t][h] (chunk rows), dR, db_nd)."""
    dev = Q.device
    h = Q.shape[-1]
    T = maxlen + t
    q = Q.to(F64).clone().requires_grad_(True)
    k = Kf.to(F64)[:, maxlen:].clone().requires_grad_(True)
    v = Vf.to(F64)[:, maxlen:].clone().requires_grad_(True)
    Rr = R.to(F64).clone().requires_grad_(True)
    bn = b_nd.to(F64).clone().requires_grad_(True)
    full_k = torch.cat([Kf.to(F64)[:, :maxlen], k], 1)
    full_v = torch.cat([Vf.to(F64)[:, :maxlen], v], 1)
    smask = None if smask_u8 is None else (smask_u8.reshape(B, 1, maxlen) != 0)
    with torch.device(dev):
        mask, _ = O.allowed_mask(first_u8[:, 0] != 0, smask, t, maxlen)
        d = (T - t + torch.arange(t)[:, None]) - torch.arange(T)[None, :]
    okb = (d >= 0) & (d < maxlen)
    D = torch.where(okb[None], bn[:, d.clamp(0, maxlen - 1)], torch.zeros((), dtype=F64, device=dev))
    Qh, Kh, Vh = O.split_heads(q.reshape(B, t, h), heads), O.split_heads(full_k, heads), O.split_heads(full_v, heads)
    Rh = O.split_heads(Rr.reshape(B, t, -1), heads)
    e = Qh.shape[2]
    bias = (~mask).to(F64).repeat_interleave(heads, dim=0) * -1e9 + torch.einsum("btn,ntp->btp", Rh, D)
    Wt = torch.softmax(torch.baddbmm(bias, Qh, Kh.transpose(-1, -2), alpha=1.0 / e), dim=2)
    A = torch.einsum("btp,bpe->bte", Wt, Vh).reshape(B, heads, t, e).permute(0, 2, 1, 3).reshape(B * t, h)
    dq, dk, dv, dR, db = torch.autograd.grad(A, (q, k, v, Rr, bn), dO.to(F64))
    return dict(dq=dq, dk=dk.reshape(B * t, h), dv=dv.reshape(B * t, h), dR=dR, db_nd=db)


def softmax_bwd(logp, idx, scale):
    """d/d logits of -scale * log_softmax(logits)[idx] = scale * (exp(logp) - onehot(idx)), float64."""
    g = torch.exp(logp.to(F64))
    g[torch.arange(g.shape[0], device=g.device), idx.long()] -= 1.0
    return g * scale


def full_attention_bwd(q, k, v, dO, B, t, heads):
    """Autograd of the IDM's unmasked attention softmax(q k^T / D) v per head (D = 128, every key of the sequence) in float64.
    q, dO [B*t][h], k, v [B, t, h] -> (dq, dk, dv) [B*t][h]."""
    h = q.shape[-1]
    D = h // heads
    split = lambda x: x.to(F64).reshape(B, t, heads, D).permute(0, 2, 1, 3)
    qq, kk, vv = (split(x).clone().requires_grad_(True) for x in (q, k, v))
    o = torch.softmax(qq @ kk.transpose(-1, -2) / D, -1) @ vv
    grads = torch.autograd.grad(o, (qq, kk, vv), split(dO))
    return [g.permute(0, 2, 1, 3).reshape(B * t, h) for g in grads]


def conv3d_t5_wgrad(img, dy, C, chunk=16):
    """Weight / bias gradient of the IDM's conv3d pre-stage (kernel (5, 1, 1), zero padding of 2 frames at both ends of each sequence)
    in float64, on the device of the inputs, `chunk` frames of dy at a time.  img u8 or fp32 [B, T, H, W, 3] on the uint8 scale, dy ZP
    [B*T, H+1, W+1, C] (the gradient wrt the conv3d output; its pad row / column is not part of the conv).  Returns (dW [C][15] in
    (dt, c) order, db [C], and the same sums over |dy|, |img|) -- dW with respect to weights that multiply the uint8-scale values."""
    B, T, H, W, _ = img.shape
    dev = dy.device
    dW, sW = torch.zeros(C, 5, 3, dtype=F64, device=dev), torch.zeros(C, 5, 3, dtype=F64, device=dev)
    db, sb = torch.zeros(C, dtype=F64, device=dev), torch.zeros(C, dtype=F64, device=dev)
    for b in range(B):
        for t0 in range(0, T, chunk):
            t1 = min(T, t0 + chunk)
            g = dy[b * T + t0:b * T + t1, :H, :W].to(F64).reshape(t1 - t0, H * W, C)
            db += g.sum((0, 1))
            sb += g.abs().sum((0, 1))
            for dt in range(5):  # output frame t reads input frame t + dt - 2
                lo, hi = max(t0, 2 - dt), min(t1, T + 2 - dt)
                if lo >= hi:
                    continue
                x = img[b, lo + dt - 2:hi + dt - 2].to(F64).reshape(hi - lo, H * W, 3)
                gg = g[lo - t0:hi - t0]
                dW[:, dt] += torch.einsum("fpo,fpc->oc", gg, x)
                sW[:, dt] += torch.einsum("fpo,fpc->oc", gg.abs(), x.abs())
    return dW.reshape(C, 15), db, sW.reshape(C, 15), sb
