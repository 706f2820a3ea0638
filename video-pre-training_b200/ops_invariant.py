"""Tensor-level wrappers of the batch-invariant mode's kernels (`MinecraftAgentPolicy.set_batch_invariant`), re-exported by `ops`; same
conventions as ops.py.  Each is its default-plan op running the launch plan of a one-row call, whatever the batch: the weight-streaming
GEMM at any M (`vpt_gemm_bf16_rowwise`), the convolution, pool and attention with a pinned plan (`vpt_*_plan`), and the Gumbel-max with
counter-based noise (`vpt_gumbel_argmax_keyed`)."""
import ctypes as C

import torch

from . import _native as nat
from . import ops


def gemm_rowwise(A, Bw, out, M, N, K, *, mr=None, rows_per_group=1, S1=None, S2=None, relu=0, out_scale=1.0, residual=None, ld_out=None, seg=None,
                 stat_part=None, stat_mode=0, dsts=None):
    """`ops.gemm` with every row computed as an M = 1 call computes it (the weight-streaming kernel over groups of 8 rows)."""
    a = ops._gemm_args(A, Bw, out, M, N, K, conv=None, mr=mr, rows_per_group=rows_per_group, S1=S1, S2=S2, relu=relu, out_scale=out_scale,
                       residual=residual, ld_out=ld_out, seg=seg, stat_part=stat_part, stat_mode=stat_mode, cluster=0, dsts=dsts)
    nat.check(nat.lib().vpt_gemm_bf16_rowwise(C.byref(a), ops._stream()), "vpt_gemm_bf16_rowwise")
    ops._count()
    return out


def conv3x3_zp_plan(x, Wb, H, W, *, mr=None, S1=None, S2=None, relu=1, residual=None, want_stats=True, out=None, Ef=None, res_scale=None,
                    res_shift=None, plan_frames=1):
    """`ops.conv3x3_zp` running the launch plan of a call of `plan_frames` frames."""
    a, out, part, P, _ = ops._conv_zp_args(x, Wb, H, W, mr, S1, S2, relu, residual, want_stats, out, Ef, res_scale, res_shift, plan_frames)
    nat.check(nat.lib().vpt_conv3x3_zp_plan(C.byref(a), plan_frames, ops._stream()), "vpt_conv3x3_zp_plan")
    ops._count()
    F_, Cout = x.shape[0], Wb.shape[0]
    return out, ops.stats_finalize(part, F_, (H + 1) * (W + 1) * P, H * W * Cout) if want_stats else None


def maxpool3s2_plan(x, zp=True, want_chan=False, plan_frames=1):
    """`ops.maxpool3s2` with the blocks (and partials) per frame of a call of `plan_frames` frames."""
    return ops._maxpool3s2(x, zp, want_chan, plan_frames)


def attention_plan(Q, Kf, Vf, R, b_nd, first_u8, smask, B, t, maxlen, heads, causal=True, plan_batch=1):
    """`ops.attention` with the long band's cluster split of a call of `plan_batch` rows."""
    return ops._attention(Q, Kf, Vf, R, b_nd, first_u8, smask, B, t, maxlen, heads, causal, plan_batch)


def gumbel_argmax_keyed(logits, keys, seed, head):
    """Gumbel-max with counter-based noise: logits fp32 [..., n] with rows = keys rows, keys device int64 [rows, 2] of (stream, step),
    seed an integer (64 bits), head the head's index -> int64 [...].  A row's pick depends on its logits and key only."""
    ops._cuda(logits, keys)
    logits = logits.contiguous()
    n = logits.shape[-1]
    rows = logits.numel() // n
    if keys.dtype != torch.int64 or tuple(keys.shape) != (rows, 2) or not keys.is_contiguous():
        raise ValueError(f"gumbel_argmax_keyed: keys must be contiguous int64 ({rows}, 2) (got {keys.dtype} {tuple(keys.shape)})")
    idx = torch.empty(logits.shape[:-1], dtype=torch.int64, device=logits.device)
    nat.check(nat.lib().vpt_gumbel_argmax_keyed(ops._p(logits), ops._p(keys), int(seed) & (2 ** 64 - 1), head, ops._p(idx), rows, n, ops._stream()),
              "vpt_gumbel_argmax_keyed")
    ops._count()
    return idx
