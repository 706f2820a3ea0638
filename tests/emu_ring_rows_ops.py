"""TEST-ONLY torch emulation of the ring-memory ops with per-environment offsets and row maps (video-pre-training_b200/ops_ring.py,
csrc/ring.cuh): `ring_write` / `attention_ring` with the optional `rows` / `row_off` and `ring_advance_rows`, same signatures and results
as the kernels.  Batch row b works on ring row rows[b] (b without `rows`), whose memory key j is at physical row
(off + row_off[r] + j) % maxlen; a row with rows[b] = -1 is inert: it writes nothing and its attention output is zero.
`attention_ring` gathers each row's keys into the linear [memory | chunk] layout and runs emu_ops.attention over all B rows at once,
as the pytree forward does."""
import torch

import emu_ops


def _rows(rows, E):
    return list(range(E)) if rows is None else [int(r) for r in rows.tolist()]


def _slot(off, row_off, r, maxlen):
    return (int(off[0]) + (0 if row_off is None else int(row_off[r]))) % maxlen


def ring_write(knew, vnew, k, v, mask, off, first_u8, rows=None, row_off=None):
    E, maxlen, h = k.shape
    rs = _rows(rows, E)
    knew, vnew = knew.reshape(len(rs), h), vnew.reshape(len(rs), h)
    for b, r in enumerate(rs):
        if r < 0:
            continue
        o = _slot(off, row_off, r, maxlen)
        k[r, o] = knew[b]
        v[r, o] = vnew[b]
        if first_u8[b, 0] != 0:
            mask[r] = False
        mask[r, o] = True


def attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads, rows=None, row_off=None):
    E, maxlen, h = k.shape
    rs = _rows(rows, E)
    B = len(rs)
    K = torch.zeros((B, maxlen + 1, h), dtype=k.dtype)
    V = torch.zeros_like(K)
    smask = torch.zeros((B, 1, maxlen), dtype=torch.uint8)
    for b, r in enumerate(rs):
        if r < 0:
            continue
        phys = (_slot(off, row_off, r, maxlen) + torch.arange(maxlen + 1)) % maxlen  # [memory | chunk] key j -> physical row
        K[b], V[b] = k[r, phys], v[r, phys]
        smask[b, 0] = mask[r, phys[:maxlen]].to(torch.uint8)
    out = emu_ops.attention(Q, K, V, R, b_nd, first_u8, smask, B, 1, maxlen, heads)
    for b, r in enumerate(rs):
        if r < 0:
            out.view(B, h)[b] = 0
    return out


def ring_advance_rows(row_off, rows, maxlen):
    for r in rows.tolist():
        if r >= 0:
            row_off[r] = (int(row_off[r]) + 1) % maxlen
