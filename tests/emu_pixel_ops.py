"""TEST-ONLY torch emulation of the image-gradient ops (video-pre-training_b200/ops_pixel.py, ops_idm.conv3d_t5_dimg), same signatures;
see emu_ops.py.  Autograd of the same forward as emu_ops.firstconv_pool, with the frames as the leaf; the temporal conv's transpose in
closed form."""
import torch
import torch.nn.functional as F

import emu_ops


def firstconv_dimg(img, w, bias, dy, C0):
    x = img.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    wt = w.reshape(C0, 3, 3, 3).permute(0, 3, 1, 2)  # [C0][ky][kx][c] -> OIHW
    y = F.max_pool2d(F.relu(F.conv2d(x, wt, bias, padding=1)), 3, 2, 1)
    (g,) = torch.autograd.grad(y, x, emu_ops.from_zp(dy).float().permute(0, 3, 1, 2))
    return g.permute(0, 2, 3, 1).contiguous()


def conv3d_t5_dimg(dy, w, B, T, H, W):
    C = w.shape[0]
    g = emu_ops.from_zp(dy).float().reshape(B, T, H, W, C)
    wt = w.reshape(C, 5, 3)  # [C][dt][c]
    out = torch.zeros((B, T, H, W, 3), dtype=torch.float32)
    for dt in range(5):  # dimg[s] += dz[s + 2 - dt] . w[dt]
        s0, s1 = max(0, dt - 2), min(T, T + dt - 2)
        if s1 > s0:
            out[:, s0:s1] += g[:, s0 + 2 - dt:s1 + 2 - dt] @ wt[:, dt, :]
    return out.reshape(B * T, H, W, 3)
