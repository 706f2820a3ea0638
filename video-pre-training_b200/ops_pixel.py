"""Tensor-level wrappers of the image-gradient kernels (csrc/firstconv_bwd.cuh, csrc/idm_bwd.cuh), re-exported by `ops`; same
conventions as ops.py."""
import torch

from . import _native as nat
from . import ops

BF16, F32 = torch.bfloat16, torch.float32


def firstconv_dimg(img, w, bias, dy, C0):
    """Image gradient of the fused first conv + ReLU + max-pool: fp32 [F,H,W,3] (uint8 scale) from dy bf16 ZP [F,H/2+1,W/2+1,C0], the
    gradient `firstconv_bwd` takes; img u8 or fp32 [F,H,W,3], w / bias the forward's (the /255-folded [C0][27] and [C0])."""
    ops._cuda(img, w, bias, dy)
    f32 = ops._frames_f32(img, "firstconv_dimg")
    F_, H, W, _ = img.shape
    if dy.dtype != BF16 or tuple(dy.shape) != (F_, H // 2 + 1, W // 2 + 1, C0) or not dy.is_contiguous():
        raise ValueError(f"firstconv_dimg: dy must be contiguous bf16 {(F_, H // 2 + 1, W // 2 + 1, C0)} (got {dy.dtype} {tuple(dy.shape)})")
    dimg = torch.empty((F_, H, W, 3), dtype=F32, device=img.device)
    nat.check(nat.lib().vpt_firstconv_dimg(ops._p(img), int(f32), ops._p(w), ops._p(bias), ops._p(dy), ops._p(dimg), F_, H, W, C0, ops._stream()), "vpt_firstconv_dimg")
    ops._count()
    return dimg


def conv3d_t5_dimg(dy, w, B, T, H, W):
    """Image gradient of `ops.conv3d_t5`: fp32 [B*T,H,W,3] (uint8 scale) from dy bf16 ZP [B*T,H+1,W+1,C] (the gradient `conv3d_t5_bwd`
    takes) and the forward's weights w fp32 [C][15] ((dt, c) order, /255-folded); zero padding in time at both ends of each sequence."""
    ops._cuda(dy, w)
    C = w.shape[0]
    if dy.dtype != BF16 or tuple(dy.shape) != (B * T, H + 1, W + 1, C) or not dy.is_contiguous():
        raise ValueError(f"conv3d_t5_dimg: dy must be contiguous bf16 {(B * T, H + 1, W + 1, C)} (got {dy.dtype} {tuple(dy.shape)})")
    if w.dtype != F32 or tuple(w.shape) != (C, 15) or not w.is_contiguous():
        raise ValueError(f"conv3d_t5_dimg: w must be contiguous fp32 [C, 15] (got {w.dtype} {tuple(w.shape)})")
    dimg = torch.empty((B * T, H, W, 3), dtype=F32, device=dy.device)
    nat.check(nat.lib().vpt_conv3d_t5_dimg(ops._p(dy), ops._p(w), ops._p(dimg), B, T, H, W, C, ops._stream()), "vpt_conv3d_t5_dimg")
    ops._count()
    return dimg

