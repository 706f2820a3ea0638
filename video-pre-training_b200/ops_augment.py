"""Tensor-level wrapper of the training-time augmentation kernel (`agent.augment_frames`, csrc/augment.cuh), re-exported by `ops`; same
conventions as ops.py."""
from . import _native as nat
from . import ops


def augment(frames, params, out):
    """u8 [F, H, W, 3] frames -> `out` (u8 or fp32, same shape): per frame the inverse affine warp and colour jitter of fp32 params [F, 10]."""
    ops._cuda(frames, params, out)
    F_, H, W, _ = frames.shape
    nat.check(nat.lib().vpt_augment_frames(ops._p(frames), ops._p(out), int(out.dtype == ops.F32), ops._p(params), F_, H, W, ops._stream()),
              "vpt_augment_frames")
    ops._count()
    return out
