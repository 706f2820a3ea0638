"""Tensor-level wrappers of the categorical heads' distribution kernels (csrc/head_dist.cuh) and of the RL head backward with the entropy
bonus (csrc/rl_bwd.cuh), re-exported by `ops`; same conventions as ops.py.  Log-probs are fp32 [rows, groups*n] with unit column stride
(any row stride), the layout the heads' forward returns."""
import torch

from . import _native as nat
from . import ops
from .ops_rl import _rows_f32

F32 = torch.float32


def _logp(name, what, t, rows=None, width=None):
    if t.dtype != F32 or t.dim() != 2 or t.stride(1) != 1 or (rows is not None and tuple(t.shape) != (rows, width)):
        want = "[rows, groups*n]" if rows is None else f"[{rows}, {width}]"
        raise ValueError(f"{name}: {what} must be fp32 {want} with unit column stride (got {t.dtype} {tuple(t.shape)})")


def _groups(name, width, groups):
    if groups <= 0 or width % groups:
        raise ValueError(f"{name}: groups = {groups} must divide the {width} columns")
    return width // groups


def head_entropy(logp, groups=1):
    """logp fp32 [rows, groups*n] -> fp32 [rows] = -sum over the row of exp(logp) * logp."""
    ops._cuda(logp)
    _logp("head_entropy", "logp", logp)
    rows, width = logp.shape
    n = _groups("head_entropy", width, groups)
    ent = torch.empty((rows,), dtype=F32, device=logp.device)
    if rows:
        nat.check(nat.lib().vpt_head_entropy(ops._p(logp), logp.stride(0), groups, n, ops._p(ent), rows, ops._stream()), "vpt_head_entropy")
        ops._count()
    return ent


def head_kl(logq, logp, groups=1):
    """logq, logp fp32 [rows, groups*n] -> fp32 [rows] = KL(q || p) = sum over the row of exp(logq) * (logq - logp)."""
    ops._cuda(logq, logp)
    _logp("head_kl", "logq", logq)
    rows, width = logq.shape
    _logp("head_kl", "logp", logp, rows, width)
    n = _groups("head_kl", width, groups)
    kl = torch.empty((rows,), dtype=F32, device=logq.device)
    if rows:
        nat.check(nat.lib().vpt_head_kl(ops._p(logq), logq.stride(0), ops._p(logp), logp.stride(0), groups, n, ops._p(kl), rows, ops._stream()),
                  "vpt_head_kl")
        ops._count()
    return kl


def head_entropy_bwd(logp, g, groups=1):
    """Backward of `head_entropy`: g fp32 [rows] (d loss / d entropy) -> fp32 [rows, groups*n] = -g * exp(logp) * (logp + 1)."""
    ops._cuda(logp, g)
    _logp("head_entropy_bwd", "logp", logp)
    rows, width = logp.shape
    n = _groups("head_entropy_bwd", width, groups)
    _rows_f32("head_entropy_bwd", "g", g, rows)
    d = torch.empty((rows, width), dtype=F32, device=logp.device)
    if rows:
        nat.check(nat.lib().vpt_head_entropy_bwd(ops._p(logp), logp.stride(0), ops._p(g), groups, n, ops._p(d), d.stride(0), rows, ops._stream()),
                  "vpt_head_entropy_bwd")
        ops._count()
    return d


def head_kl_bwd(logq, logp, g, groups=1, want_q=True, want_p=True):
    """Backward of `head_kl`: g fp32 [rows] -> (d logq, d logp) fp32 [rows, groups*n] = (g * exp(logq) * (logq - logp + 1), -g * exp(logq));
    a side not wanted is None and is not computed."""
    ops._cuda(logq, logp, g)
    _logp("head_kl_bwd", "logq", logq)
    rows, width = logq.shape
    _logp("head_kl_bwd", "logp", logp, rows, width)
    n = _groups("head_kl_bwd", width, groups)
    _rows_f32("head_kl_bwd", "g", g, rows)
    dq = torch.empty((rows, width), dtype=F32, device=logq.device) if want_q else None
    dp = torch.empty((rows, width), dtype=F32, device=logq.device) if want_p else None
    if rows and (want_q or want_p):
        nat.check(nat.lib().vpt_head_kl_bwd(ops._p(logq), logq.stride(0), ops._p(logp), logp.stride(0), ops._p(g), groups, n, ops._p(dq),
                                            width, ops._p(dp), width, rows, ops._stream()), "vpt_head_kl_bwd")
        ops._count()
    return dq, dp


def rl_head_bwd_ent(logp, idx, c, logq, k, e, inv_temp, out, col0, kl=None, ent=None):
    """`ops.rl_head_bwd` with the entropy bonus: adds e * exp(logp) * (logp + H) * inv_temp to the head's columns of `out` (e = ent_coef / N,
    the gradient of -ent_coef * mean H; nothing is added when e == 0, and `out` then holds `rl_head_bwd`'s bits) and returns (kl, ent) fp32
    [rows], ent = H = -sum exp(logp) * logp per row (each added to the given tensor when one is passed)."""
    ops._cuda(logp, idx, c, logq, out, kl, ent)
    if logp.dtype != F32 or logp.dim() != 2 or logp.stride(1) != 1:
        raise ValueError("rl_head_bwd_ent: logp must be fp32 [rows, n] with unit column stride")
    rows, n = logp.shape
    if logq is not None and (logq.dtype != F32 or tuple(logq.shape) != (rows, n) or logq.stride(1) != 1):
        raise ValueError(f"rl_head_bwd_ent: logq must be fp32 [{rows}, {n}] with unit column stride")
    if idx.dtype != torch.int64 or idx.numel() != rows or not idx.is_contiguous():
        raise ValueError(f"rl_head_bwd_ent: idx must be contiguous int64 with {rows} elements")
    _rows_f32("rl_head_bwd_ent", "c", c, rows)
    if out.dtype != torch.bfloat16 or out.dim() != 2 or out.shape[0] != rows or out.shape[1] < col0 + n or col0 < 0 or out.stride(1) != 1:
        raise ValueError("rl_head_bwd_ent: out must be bf16 [rows, >= col0 + n] with unit column stride")
    if rows and (int(idx.min()) < 0 or int(idx.max()) >= n):  # (one host sync: the kernel would index past the head's columns)
        raise ValueError(f"rl_head_bwd_ent: actions must lie in [0, {n})")
    if (kl is None) != (ent is None):
        raise ValueError("rl_head_bwd_ent: pass both kl and ent to accumulate into, or neither")
    acc = kl is not None
    if acc:
        _rows_f32("rl_head_bwd_ent", "kl", kl, rows)
        _rows_f32("rl_head_bwd_ent", "ent", ent, rows)
    else:
        kl = torch.empty((rows,), dtype=F32, device=logp.device)
        ent = torch.empty((rows,), dtype=F32, device=logp.device)
    nat.check(nat.lib().vpt_rl_head_bwd_ent(ops._p(logp), logp.stride(0), ops._p(logq), 0 if logq is None else logq.stride(0), ops._p(idx),
                                            ops._p(c), float(k), float(e), float(inv_temp), n, ops._p(out), out.stride(0), col0, ops._p(kl),
                                            ops._p(ent), int(acc), rows, ops._stream()), "vpt_rl_head_bwd_ent")
    ops._count()
    return kl, ent
