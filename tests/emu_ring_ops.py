"""TEST-ONLY torch emulation of the ring-memory ops (video-pre-training_b200/ops_ring.py, csrc/ring.cuh): same signatures, same results as
the kernels.  `attention_ring` gathers the ring's rows into the linear [memory | chunk] layout and runs emu_ops.attention on it, which is
what the kernel's row addressing promises."""
import torch

import emu_ops


def ring_write(knew, vnew, k, v, mask, off, first_u8):
    B, maxlen, h = k.shape
    o = int(off[0])
    k[:, o] = knew.reshape(B, h)
    v[:, o] = vnew.reshape(B, h)
    mask[first_u8[:, 0] != 0] = False
    mask[:, o] = True


def attention_ring(Q, k, v, R, b_nd, first_u8, mask, off, heads):
    B, maxlen, h = k.shape
    rows = (int(off[0]) + torch.arange(maxlen + 1)) % maxlen  # [memory | chunk] key j -> ring row
    smask = mask[:, rows[:maxlen]].to(torch.uint8).reshape(B, 1, maxlen)
    return emu_ops.attention(Q, k[:, rows], v[:, rows], R, b_nd, first_u8, smask, B, 1, maxlen, heads)


def ring_advance(off, maxlen):
    off.copy_((off + 1) % maxlen)
