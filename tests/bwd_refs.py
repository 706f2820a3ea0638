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
def backward_shapes(width, B=16, T=128):
    """The call shapes the BC backward (training.py) reaches for `policy_kwargs(width)` at B x T frames / tokens."""
    cfg = NetConfig(**vpt_b200.policy_kwargs(width))
    H0, W0, _ = cfg.img_shape
    c = cfg.chans
    h, heads = cfg.hidsize, cfg.heads
    Hf, Wf = cfg.final_hw
    kd = (Hf + 1) * (Wf + 1) * c[-1]                 # dense input row in ZP (h, w, c) order
    kcat = (3 * h + NBASIS * heads + 7) // 8 * 8      # q | k | v | R gradient buffer (training.py)
    heads_n = [(name, sp.eltype.n) for name, sp in vpt_b200.minecraft_action_space().items()]
    cols, c0 = [], 0
    for name, n in heads_n:
        cols.append((name, c0, n))
        c0 += n
    ld_logits = (c0 + 7) // 8 * 8
    # 3x3 convs of the CNN backward, (H, W, Cin, Cout) at their frame size: stack i > 0 opens with a conv at the previous size
    convs, norms, pools = [], [], []
    Hs, Ws = H0 // 2, W0 // 2
    for i, C in enumerate(c):
        if i > 0:
            convs.append((Hs, Ws, c[i - 1], C))
            pools.append((Hs, Ws, C))                    # max-pool backward input (pre-pool size)
            Hs, Ws = Hs // 2, Ws // 2
        convs.append((Hs, Ws, C, C))
        norms.append((Hs, Ws, C))                        # GroupNorm(1) ZP frames of this stack
    assert (Hs, Ws) == (Hf, Wf)
    uniq = lambda v: list(dict.fromkeys(v))
    return dict(
        cfg=cfg, B=B, T=T, N=B * T, h=h, heads=heads, maxlen=cfg.maxlen, kcat=kcat, ld_logits=ld_logits, head_cols=cols,
        convs=uniq(convs), gn=uniq(norms), pools=uniq(pools), firstconv=(H0, W0, c[0]),
        ln=uniq([h, cfg.cnn_outsize]), dense=(Hf, Wf, c[-1], kd),
        linears=uniq([(ld_logits, h), (kcat, h), (h, h * cfg.pointwise_ratio), (h * cfg.pointwise_ratio, h), (h, h),
                      (h, cfg.cnn_outsize), (cfg.cnn_outsize, kd)]),
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


def norm_bwd(du, x, gamma, rows_per_group, zp=None):
    """Autograd of GroupNorm(1) over a ZP frame (rows_per_group > 1) or LayerNorm over a row (rows_per_group == 1; with zp the row
    is a ZP image whose pads are not part of the norm) in float64.  gamma: fp32 [C].
    Returns dict(dx [rows][C] (zero at pads), dgamma [C], dbeta [C], ms [G][2] = (mean gamma*du, mean gamma*du*n))."""
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
