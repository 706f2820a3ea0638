"""Tensor-level wrappers of the ring-memory kernels (csrc/ring.cuh, `vpt_attention_ring`), re-exported by `ops`; same conventions as ops.py.
A ring holds a layer's KV memory as K / V bf16 [E, maxlen, h] and the state mask u8 [E, maxlen] with memory key j of ring row e at row
(off + row_off[e] + j) % maxlen; `off` is a device int32 [1] and `row_off` None (all zeros) or a device int32 [E] (policy.py RingState).
A step of some of the rows passes `rows`, int32 [B]: batch row b is ring row rows[b], or an inert padding row where rows[b] = -1."""
import torch

from . import _native as nat
from . import ops

BF16 = torch.bfloat16


def _ring(name, k, v, mask, off, E, maxlen, h):
    if k.dtype != BF16 or v.dtype != BF16 or tuple(k.shape) != (E, maxlen, h) or v.shape != k.shape or not (k.is_contiguous() and v.is_contiguous()):
        raise ValueError(f"{name}: the ring's K / V must be contiguous bf16 {(E, maxlen, h)} (got {k.dtype} {tuple(k.shape)}, {v.dtype} {tuple(v.shape)})")
    if mask.dtype not in (torch.uint8, torch.bool) or tuple(mask.shape) != (E, maxlen) or not mask.is_contiguous():
        raise ValueError(f"{name}: the ring's mask must be contiguous uint8 / bool {(E, maxlen)} (got {mask.dtype} {tuple(mask.shape)})")
    if off.dtype != torch.int32 or off.numel() != 1:
        raise ValueError(f"{name}: the ring offset must be one int32 (got {off.dtype} {tuple(off.shape)})")


def _rows(name, rows, row_off, E):
    """The step's batch size: len(rows), or E for a step of every row."""
    if row_off is not None and (row_off.dtype != torch.int32 or tuple(row_off.shape) != (E,) or not row_off.is_contiguous()):
        raise ValueError(f"{name}: row_off must be contiguous int32 ({E},) (got {row_off.dtype} {tuple(row_off.shape)})")
    if rows is None:
        return E
    if rows.dtype != torch.int32 or rows.dim() != 1 or rows.numel() == 0 or not rows.is_contiguous():
        raise ValueError(f"{name}: rows must be a non-empty contiguous int32 vector (got {rows.dtype} {tuple(rows.shape)})")
    return rows.numel()


def ring_write(knew, vnew, k, v, mask, off, first_u8, rows=None, row_off=None):
    """The step's K / V rows knew, vnew bf16 [B, h] (or [B, 1, h]) -> the slot (off + row_off[r]) % maxlen of ring row r = rows[b] (r = b
    without `rows`; inert rows write nothing); mask[r, slot] = 1 and, for every b with first_u8[b, 0], the rest of mask[r] = 0."""
    ops._cuda(knew, vnew, k, v, mask, off, first_u8, rows, row_off)
    E, maxlen, h = k.shape
    _ring("ring_write", k, v, mask, off, E, maxlen, h)
    B = _rows("ring_write", rows, row_off, E)
    for name, x in (("knew", knew), ("vnew", vnew)):
        if x.dtype != BF16 or x.numel() != B * h or not x.is_contiguous():
            raise ValueError(f"ring_write: {name} must be contiguous bf16 with {B} rows of {h} (got {x.dtype} {tuple(x.shape)})")
    if rows is None and row_off is None:
        nat.check(nat.lib().vpt_ring_write(ops._p(knew), ops._p(vnew), ops._p(k), ops._p(v), ops._p(mask), ops._p(first_u8), first_u8.stride(0),
                                           ops._p(off), B, maxlen, h, ops._stream()), "vpt_ring_write")
    else:
        nat.check(nat.lib().vpt_ring_write_rows(ops._p(knew), ops._p(vnew), ops._p(k), ops._p(v), ops._p(mask), ops._p(first_u8), first_u8.stride(0),
                                                ops._p(off), ops._p(rows), ops._p(row_off), B, maxlen, h, ops._stream()), "vpt_ring_write_rows")
    ops._count()


def attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads, rows=None, row_off=None):
    """`ops.attention` (causal, t = 1) with the KV memory and the step's own row read from the ring (after `ring_write`): Q bf16 [B, h].
    With `rows`, batch row b (Q, R, first, out) attends over ring row rows[b]; an inert row's output is zero."""
    return _attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads, rows, row_off, None)


def attention_ring_plan(Q, k, v, R, b_nd, first_u8, mask, off, heads, rows=None, row_off=None, plan_batch=1):
    """`attention_ring` with the long band's cluster split of a call of `plan_batch` rows (the batch-invariant mode)."""
    return _attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads, rows, row_off, plan_batch)


def _attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads, rows, row_off, plan_batch):
    ops._cuda(Q, k, v, R, b_nd, first_u8, mask, off, rows, row_off)
    E, maxlen, h = k.shape
    _ring("attention_ring", k, v, mask, off, E, maxlen, h)
    B = _rows("attention_ring", rows, row_off, E)
    if Q.dtype != BF16 or Q.numel() != B * h or not Q.is_contiguous():
        raise ValueError(f"attention_ring: Q must be contiguous bf16 with {B} rows of {h} (one step; got {Q.dtype} {tuple(Q.shape)})")
    out = torch.empty_like(Q)
    if plan_batch is not None and rows is None and row_off is None:
        nat.check(nat.lib().vpt_attention_ring_plan(ops._p(Q), ops._p(k), ops._p(v), ops._p(R), R.stride(-2), ops._p(b_nd), ops._p(first_u8),
                                                    first_u8.stride(0), ops._p(mask), ops._p(off), ops._p(out), B, maxlen, heads, b_nd.shape[0],
                                                    plan_batch, ops._stream()), "vpt_attention_ring_plan")
    elif plan_batch is not None:
        nat.check(nat.lib().vpt_attention_ring_rows_plan(ops._p(Q), ops._p(k), ops._p(v), ops._p(R), R.stride(-2), ops._p(b_nd), ops._p(first_u8),
                                                         first_u8.stride(0), ops._p(mask), ops._p(off), ops._p(rows), ops._p(row_off), ops._p(out),
                                                         B, maxlen, heads, b_nd.shape[0], plan_batch, ops._stream()), "vpt_attention_ring_rows_plan")
    elif rows is None and row_off is None:
        nat.check(nat.lib().vpt_attention_ring(ops._p(Q), ops._p(k), ops._p(v), ops._p(R), R.stride(-2), ops._p(b_nd), ops._p(first_u8),
                                               first_u8.stride(0), ops._p(mask), ops._p(off), ops._p(out), B, maxlen, heads, b_nd.shape[0],
                                               ops._stream()), "vpt_attention_ring")
    else:
        nat.check(nat.lib().vpt_attention_ring_rows(ops._p(Q), ops._p(k), ops._p(v), ops._p(R), R.stride(-2), ops._p(b_nd), ops._p(first_u8),
                                                    first_u8.stride(0), ops._p(mask), ops._p(off), ops._p(rows), ops._p(row_off), ops._p(out), B,
                                                    maxlen, heads, b_nd.shape[0], ops._stream()), "vpt_attention_ring_rows")
    ops._count()
    return out


def ring_advance(off, maxlen):
    """off = (off + 1) % maxlen on the device: the step's rows become the newest memory rows."""
    ops._cuda(off)
    nat.check(nat.lib().vpt_ring_advance(ops._p(off), maxlen, ops._stream()), "vpt_ring_advance")
    ops._count()


def ring_advance_rows(row_off, rows, maxlen):
    """row_off[r] = (row_off[r] + 1) % maxlen on the device for every ring row r in `rows` (-1 entries skipped): the end of a step of
    those rows only, which leaves `off` and every other row where they are."""
    ops._cuda(row_off, rows)
    _rows("ring_advance_rows", rows, None, 0)
    if row_off.dtype != torch.int32 or row_off.dim() != 1 or not row_off.is_contiguous():
        raise ValueError(f"ring_advance_rows: row_off must be a contiguous int32 vector (got {row_off.dtype} {tuple(row_off.shape)})")
    nat.check(nat.lib().vpt_ring_advance_rows(ops._p(row_off), ops._p(rows), rows.numel(), maxlen, ops._stream()), "vpt_ring_advance_rows")
    ops._count()


def ring_noise_keys(steps, rows, B):
    """The sampling keys of a step of B batch rows (batch-invariant mode): int64 [B, 2], row b = (r, steps[r]) for its environment r =
    rows[b] (r = b without `rows`), then steps[r] += 1 on the device; an inert row (rows[b] = -1) gets (-1, 0) and advances nothing."""
    ops._cuda(steps, rows)
    if steps.dtype != torch.int64 or steps.dim() != 1 or not steps.is_contiguous():
        raise ValueError(f"ring_noise_keys: steps must be a contiguous int64 vector (got {steps.dtype} {tuple(steps.shape)})")
    if rows is not None:
        B = _rows("ring_noise_keys", rows, None, 0)
    keys = torch.empty((B, 2), dtype=torch.int64, device=steps.device)
    nat.check(nat.lib().vpt_ring_noise_keys(ops._p(steps), ops._p(rows), ops._p(keys), B, ops._stream()), "vpt_ring_noise_keys")
    ops._count()
    return keys
