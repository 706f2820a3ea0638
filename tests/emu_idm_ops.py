"""TEST-ONLY torch emulation of the IDM backward ops (video-pre-training_b200/ops_idm.py), same signatures; see emu_ops.py."""
import torch
import torch.nn.functional as F

import emu_ops

F32 = torch.float32


def conv3d_t5_bwd(img, dy, C):
    """(dW fp32 [C][15] in (dt, c) order for the /255-scaled weights, db [C]) by float64 autograd of the conv3d (before its ReLU: dy is
    masked)."""
    B, T, H, W, _ = img.shape
    x = img.double().permute(0, 4, 1, 2, 3)                                    # b c t h w
    w = torch.zeros(C, 3, 5, 1, 1, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(C, dtype=torch.float64, requires_grad=True)
    y = F.conv3d(x, w, b, padding=(2, 0, 0))                                   # per-sample zero padding in time
    g = emu_ops.from_zp(dy).double().reshape(B, T, H, W, C).permute(0, 4, 1, 2, 3)
    gw, gb = torch.autograd.grad(y, (w, b), g)
    return gw.reshape(C, 3, 5).permute(0, 2, 1).reshape(C, 15).to(F32).contiguous(), gb.to(F32)


def softmax_nll_bwd_grouped(logp, idx, scale, out, col0, lp=None):
    rows, groups, n = logp.shape
    p = torch.exp(logp.float())
    p.scatter_add_(-1, idx.long().unsqueeze(-1), -torch.ones(rows, groups, 1))
    out[:, col0:col0 + groups * n] = (p * scale).reshape(rows, groups * n).to(out.dtype)
    r = logp.gather(-1, idx.long().unsqueeze(-1)).squeeze(-1).sum(-1)
    return r if lp is None else lp + r
