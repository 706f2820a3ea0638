"""TEST-ONLY torch emulation of the differentiable forward's op (video-pre-training_b200/ops_autograd.py), same signature; see emu_ops.py."""
import torch

F32 = torch.float32


def log_softmax_bwd(logp, g, scale, out, col0, groups=1, mask=None):
    rows, width = logp.shape
    n = width // groups
    lp, gg = logp.float().reshape(rows, groups, n), g.float().reshape(rows, groups, n)
    d = scale * (gg - torch.exp(lp) * gg.sum(-1, keepdim=True))
    d = d.reshape(rows, width)
    if mask is not None:
        d = torch.where(mask.bool(), d, torch.zeros((), dtype=F32))
    out[:, col0:col0 + width] = d.to(out.dtype)
    return out
