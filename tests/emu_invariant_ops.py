"""TEST-ONLY emulation of the batch-invariant mode's ops (video-pre-training_b200/ops_invariant.py, ops_ring.py; csrc/gemv_small.cuh,
conv_zp.cuh, elementwise.cuh, attention.cuh, heads.cuh, ring.cuh), same signatures: the row-wise GEMM and the pinned-plan convolution, pool
and attention return the default emulated ops' results (the emulation has no launch plan), `ring_noise_keys` builds the keys and advances the counters as the kernel does,
and `gumbel_argmax_keyed` draws from `philox4x32_10`, a numpy Philox4x32-10 (Salmon et al., SC 2011)."""
import numpy as np
import torch

import emu_ops
import emu_ring_rows_ops

_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_W = (np.uint32(0x9E3779B9), np.uint32(0xBB67AE85))


def philox4x32_10(ctr, key):
    """ctr uint32 (..., 4), key uint32 (..., 2) -> uint32 (..., 4): ten Philox4x32 rounds."""
    c = [np.asarray(ctr, dtype=np.uint32)[..., i].astype(np.uint64) for i in range(4)]
    k = [np.asarray(key, dtype=np.uint32)[..., i].astype(np.uint64) for i in range(2)]
    mask = np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r > 0:
            k = [(k[0] + np.uint64(_W[0])) & mask, (k[1] + np.uint64(_W[1])) & mask]
        p0, p1 = _M[0] * c[0], _M[1] * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & mask, p1 >> np.uint64(32), p1 & mask
        c = [hi1 ^ c[1] ^ k[0], lo1, hi0 ^ c[3] ^ k[1], lo0]
    return np.stack(c, -1).astype(np.uint32)


def keyed_uniforms(keys, seed, head, n):
    """The uniforms of `vpt_gumbel_argmax_keyed`: fp32 (rows, n) for keys int64 (rows, 2) of (stream, step)."""
    keys = np.asarray(keys, dtype=np.int64)
    rows = keys.shape[0]
    j = np.arange(n)
    ctr = np.zeros((rows, n, 4), dtype=np.uint32)
    ctr[..., 0] = j // 4
    ctr[..., 1] = head
    ctr[..., 2] = (keys[:, 0:1] & 0xFFFFFFFF).astype(np.uint32)
    ctr[..., 3] = (keys[:, 1:2] & 0xFFFFFFFF).astype(np.uint32)
    seed = int(seed) & (2 ** 64 - 1)
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32)
    words = philox4x32_10(ctr, np.broadcast_to(key, (rows, n, 2)))
    x = np.take_along_axis(words, (j % 4)[None, :, None].repeat(rows, 0), -1)[..., 0]
    return (((x >> 9).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)).astype(np.float32)


def keyed_scores(logits, keys, seed, head):
    """fp32 numpy (rows, n): logit - log(-log u)."""
    lg = logits.detach().cpu().reshape(-1, logits.shape[-1]).float().numpy()
    u = keyed_uniforms(keys.cpu().numpy(), seed, head, lg.shape[1])
    return (lg - np.log(-np.log(u))).astype(np.float32)


def gumbel_argmax_keyed(logits, keys, seed, head):
    n = logits.shape[-1]
    rows = logits.numel() // n
    if keys.dtype != torch.int64 or tuple(keys.shape) != (rows, 2):
        raise ValueError(f"gumbel_argmax_keyed: keys must be int64 ({rows}, 2) (got {keys.dtype} {tuple(keys.shape)})")
    idx = keyed_scores(logits, keys, seed, head).argmax(1)  # (numpy argmax: the lowest index of a tie)
    return torch.as_tensor(idx, dtype=torch.int64).reshape(logits.shape[:-1])


def ring_noise_keys(steps, rows, B):
    rs = list(range(B)) if rows is None else [int(r) for r in rows.tolist()]
    keys = torch.empty((len(rs), 2), dtype=torch.int64)
    for b, r in enumerate(rs):
        if r < 0:
            keys[b] = torch.tensor([-1, 0])
            continue
        keys[b] = torch.tensor([r, int(steps[r])])
        steps[r] += 1
    return keys


def gemm_rowwise(A, Bw, out, M, N, K, **kw):
    return emu_ops.gemm(A, Bw, out, M, N, K, **kw)


def conv3x3_zp_plan(x, Wb, H, W, *, plan_frames=1, **kw):
    return emu_ops.conv3x3_zp(x, Wb, H, W, **kw)


def maxpool3s2_plan(x, zp=True, want_chan=False, plan_frames=1):
    return emu_ops.maxpool3s2(x, zp, want_chan)


def attention_plan(*args, plan_batch=1, **kw):
    return emu_ops.attention(*args, **kw)


def attention_ring_plan(*args, plan_batch=1, **kw):
    return emu_ring_rows_ops.attention_ring(*args, **kw)
