"""Tensor-level wrappers of the ring-memory kernels (csrc/ring.cuh, `vpt_attention_ring`), re-exported by `ops`; same conventions as ops.py.
A ring holds a layer's KV memory as K / V bf16 [B, maxlen, h] and the state mask u8 [B, maxlen] with memory key j at row (off + j) % maxlen;
`off` is a device int32 [1] (policy.py RingState)."""
import torch

from . import _native as nat
from . import ops

BF16 = torch.bfloat16


def _ring(name, k, v, mask, off, B, maxlen, h):
    if k.dtype != BF16 or v.dtype != BF16 or tuple(k.shape) != (B, maxlen, h) or v.shape != k.shape or not (k.is_contiguous() and v.is_contiguous()):
        raise ValueError(f"{name}: the ring's K / V must be contiguous bf16 {(B, maxlen, h)} (got {k.dtype} {tuple(k.shape)}, {v.dtype} {tuple(v.shape)})")
    if mask.dtype not in (torch.uint8, torch.bool) or tuple(mask.shape) != (B, maxlen) or not mask.is_contiguous():
        raise ValueError(f"{name}: the ring's mask must be contiguous uint8 / bool {(B, maxlen)} (got {mask.dtype} {tuple(mask.shape)})")
    if off.dtype != torch.int32 or off.numel() != 1:
        raise ValueError(f"{name}: the ring offset must be one int32 (got {off.dtype} {tuple(off.shape)})")


def ring_write(knew, vnew, k, v, mask, off, first_u8):
    """The step's K / V rows knew, vnew bf16 [B, h] (or [B, 1, h]) -> ring row `off` of k / v; mask[:, off] = 1 and, for every b with
    first_u8[b, 0], the rest of mask[b] = 0."""
    ops._cuda(knew, vnew, k, v, mask, off, first_u8)
    B, maxlen, h = k.shape
    _ring("ring_write", k, v, mask, off, B, maxlen, h)
    for name, x in (("knew", knew), ("vnew", vnew)):
        if x.dtype != BF16 or x.numel() != B * h or not x.is_contiguous():
            raise ValueError(f"ring_write: {name} must be contiguous bf16 with {B} rows of {h} (got {x.dtype} {tuple(x.shape)})")
    nat.check(nat.lib().vpt_ring_write(ops._p(knew), ops._p(vnew), ops._p(k), ops._p(v), ops._p(mask), ops._p(first_u8), first_u8.stride(0), ops._p(off),
                                       B, maxlen, h, ops._stream()), "vpt_ring_write")
    ops._count()


def attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads):
    """`ops.attention` (causal, t = 1) with the KV memory and the step's own row read from the ring (after `ring_write`): Q bf16 [B, h]."""
    ops._cuda(Q, k, v, R, b_nd, first_u8, mask, off)
    B, maxlen, h = k.shape
    _ring("attention_ring", k, v, mask, off, B, maxlen, h)
    if Q.dtype != BF16 or Q.numel() != B * h or not Q.is_contiguous():
        raise ValueError(f"attention_ring: Q must be contiguous bf16 with {B} rows of {h} (one step; got {Q.dtype} {tuple(Q.shape)})")
    out = torch.empty_like(Q)
    nat.check(nat.lib().vpt_attention_ring(ops._p(Q), ops._p(k), ops._p(v), ops._p(R), R.stride(-2), ops._p(b_nd), ops._p(first_u8), first_u8.stride(0),
                                           ops._p(mask), ops._p(off), ops._p(out), B, maxlen, heads, b_nd.shape[0], ops._stream()), "vpt_attention_ring")
    ops._count()
    return out


def ring_advance(off, maxlen):
    """off = (off + 1) % maxlen on the device: the step's rows become the newest memory rows."""
    ops._cuda(off)
    nat.check(nat.lib().vpt_ring_advance(ops._p(off), maxlen, ops._stream()), "vpt_ring_advance")
    ops._count()
