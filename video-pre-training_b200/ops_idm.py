"""Tensor-level wrappers of the IDM backward kernels (csrc/idm_bwd.cuh), re-exported by `ops`; same conventions as ops.py."""
import torch

from . import _native as nat
from . import ops

F32 = torch.float32


def conv3d_t5_bwd(img, dy, C):
    """Weight / bias gradient of `ops.conv3d_t5`: img u8 or fp32 [B,T,H,W,3], dy bf16 ZP [B*T,H+1,W+1,C] = gradient wrt the conv3d output
    with its ReLU mask already applied -> (dW fp32 [C][15] in (dt, c) order for the /255-scaled kernel weights, db fp32 [C])."""
    ops._cuda(img, dy)
    if img.dtype not in (torch.uint8, F32) or img.dim() != 5 or img.shape[-1] != 3 or not img.is_contiguous():
        raise ValueError(f"conv3d_t5_bwd: img must be contiguous u8 or fp32 [B,T,H,W,3] (got {img.dtype} {tuple(img.shape)})")
    B, T, H, W, _ = img.shape
    if dy.dtype != torch.bfloat16 or tuple(dy.shape) != (B * T, H + 1, W + 1, C) or not dy.is_contiguous():
        raise ValueError(f"conv3d_t5_bwd: dy must be contiguous bf16 {(B * T, H + 1, W + 1, C)} (got {dy.dtype} {tuple(dy.shape)})")
    ws = torch.empty((max(nat.lib().vpt_conv3d_t5_bwd_workspace(B * T, H, W, C), 1),), dtype=F32, device=img.device)
    dW = torch.empty((C, 15), dtype=F32, device=img.device)
    db = torch.empty((C,), dtype=F32, device=img.device)
    fn = "vpt_conv3d_t5_bwd_f32" if img.dtype == F32 else "vpt_conv3d_t5_bwd"
    nat.check(getattr(nat.lib(), fn)(ops._p(img), ops._p(dy), ops._p(dW), ops._p(db), ops._p(ws), B, T, H, W, C, ops._stream()), fn)
    ops._count(2)
    return dW, db


def softmax_nll_bwd_grouped(logp, idx, scale, out, col0, lp=None):
    """Factored categorical head: logp fp32 [rows, groups, n] (log-softmax of every group), idx int64 [rows, groups] ->
    out[:, col0 + g*n + j] = (exp(logp) - onehot(idx)) * scale (bf16); returns lp fp32 [rows] = sum over the groups of the taken
    sub-actions' log-probs (added to `lp` when given)."""
    ops._cuda(logp, idx, out, lp)
    rows, groups, n = logp.shape
    if logp.dtype != F32 or logp.stride(2) != 1 or logp.stride(1) != n:
        raise ValueError("softmax_nll_bwd_grouped: logp must be fp32 [rows, groups, n] with the groups side by side in a row")
    if tuple(idx.shape) != (rows, groups):
        raise ValueError(f"softmax_nll_bwd_grouped: idx must be [rows, groups] = {(rows, groups)} (got {tuple(idx.shape)})")
    if out.dtype != torch.bfloat16 or out.shape[0] != rows or out.shape[1] < col0 + groups * n or out.stride(1) != 1:
        raise ValueError("softmax_nll_bwd_grouped: out must be bf16 [rows, >= col0 + groups*n] with unit column stride")
    idx = idx.to(torch.int64).contiguous()
    if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= n):  # (one host sync: the kernel would read logp out of bounds)
        raise ValueError(f"softmax_nll_bwd_grouped: actions must lie in [0, {n})")
    if lp is not None and (lp.dtype != F32 or tuple(lp.shape) != (rows,) or not lp.is_contiguous()):
        raise ValueError(f"softmax_nll_bwd_grouped: lp must be contiguous fp32 [{rows}]")
    acc = lp is not None
    if lp is None:
        lp = torch.empty((rows,), dtype=F32, device=logp.device)
    nat.check(nat.lib().vpt_softmax_nll_bwd_grouped(ops._p(logp), logp.stride(0), ops._p(idx), groups, n, float(scale), ops._p(out), out.stride(0), col0,
                                                    ops._p(lp), int(acc), rows, ops._stream()), "vpt_softmax_nll_bwd_grouped")
    ops._count()
    return lp
