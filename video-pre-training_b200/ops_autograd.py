"""Tensor-level wrapper of the differentiable forward's head backward (csrc/log_softmax_bwd.cuh), re-exported by `ops`; same conventions
as ops.py."""
import torch

from . import _native as nat
from . import ops

F32 = torch.float32


def log_softmax_bwd(logp, g, scale, out, col0, groups=1, mask=None):
    """Backward of logp = log_softmax(logits * scale) over each of `groups` groups of n columns: logp, g fp32 [rows, groups*n] (g = d loss /
    d logp), mask None or bool / uint8 [rows, groups*n] (False = the logit was masked out) ->
    out[:, col0 + k*n + j] = scale * (g - exp(logp) * sum_j g) per group, 0 where masked (bf16)."""
    ops._cuda(logp, g, out, mask)
    if logp.dtype != F32 or logp.dim() != 2 or logp.stride(1) != 1:
        raise ValueError("log_softmax_bwd: logp must be fp32 [rows, groups*n] with unit column stride")
    rows, width = logp.shape
    if groups <= 0 or width % groups:
        raise ValueError(f"log_softmax_bwd: groups = {groups} must divide the {width} columns")
    n = width // groups
    if g.dtype != F32 or tuple(g.shape) != (rows, width) or g.stride(1) != 1:
        raise ValueError(f"log_softmax_bwd: g must be fp32 [{rows}, {width}] with unit column stride")
    if out.dtype != torch.bfloat16 or out.dim() != 2 or out.shape[0] != rows or col0 < 0 or out.shape[1] < col0 + width or out.stride(1) != 1:
        raise ValueError(f"log_softmax_bwd: out must be bf16 [{rows}, >= col0 + {width}] with unit column stride")
    if mask is not None:
        if mask.dtype not in (torch.bool, torch.uint8) or tuple(mask.shape) != (rows, width) or not mask.is_contiguous():
            raise ValueError(f"log_softmax_bwd: mask must be contiguous bool / uint8 [{rows}, {width}]")
        mask = mask.view(torch.uint8)
    if rows == 0:
        return out
    nat.check(nat.lib().vpt_log_softmax_bwd(ops._p(logp), logp.stride(0), ops._p(g), g.stride(0), ops._p(mask), groups, n, float(scale), ops._p(out),
                                            out.stride(0), col0, rows, ops._stream()), "vpt_log_softmax_bwd")
    ops._count()
    return out
