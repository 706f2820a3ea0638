"""float64 closed forms of the two image-gradient kernels (csrc/firstconv_bwd.cuh vpt_firstconv_dimg, csrc/idm_bwd.cuh
vpt_conv3d_t5_dimg), for tests/test_gpu_pixel_grad.py.  They run wherever their inputs are (the GPU test keeps them on the device)."""
import torch
import torch.nn.functional as F


def from_zp(x):
    return x[:, :-1, :-1, :]


def routed(img, w, bias, dy, C0):
    """(x, dpre): the frames as float64 NCHW and the pooled gradient routed to the first positive maximum of each window, float64."""
    x = img.double().permute(0, 3, 1, 2)
    wt = w.double().reshape(C0, 3, 3, 3).permute(0, 3, 1, 2)
    pre = F.conv2d(x, wt, bias.double(), padding=1).requires_grad_(True)
    y = F.max_pool2d(F.relu(pre), 3, 2, 1)
    (dpre,) = torch.autograd.grad(y, pre, from_zp(dy).double().permute(0, 3, 1, 2))
    return x, dpre


def firstconv_dimg(img, w, bias, dy, C0):
    """d loss / d img [F, H, W, 3] = the routed gradient contracted with w over the 3x3 taps (conv_transpose2d), float64."""
    _, dpre = routed(img, w, bias, dy, C0)
    wt = w.double().reshape(C0, 3, 3, 3).permute(0, 3, 1, 2)
    return F.conv_transpose2d(dpre, wt, padding=1).permute(0, 2, 3, 1)


def conv3d_t5_dimg(dy, w, B, T, H, W):
    """dimg[b, s] = sum_dt dy[b, s + 2 - dt] . w[dt] (zero outside [0, T)) -> [B*T, H, W, 3] float64, one frame at a time."""
    C = w.shape[0]
    wt = w.double().reshape(C, 5, 3)
    g = from_zp(dy).reshape(B, T, H, W, C)
    out = torch.zeros((B, T, H, W, 3), dtype=torch.float64, device=dy.device)
    for s in range(T):
        for dt in range(5):
            t = s + 2 - dt
            if 0 <= t < T:
                out[:, s] += g[:, t].double() @ wt[:, dt, :]
    return out.reshape(B * T, H, W, 3)
