"""TEST-ONLY torch emulation of the attention backward through the KV memory (video-pre-training_b200/ops_bptt.py), same signature; see
emu_ops.py.  Autograd of the same attention as emu_ops.attention_bwd, with the memory rows of K / V as leaves too."""
import torch

import emu_ops


def attention_bwd_state(Q, Kf, Vf, R, b_nd, first_u8, smask, dO, out, B, t, maxlen, heads, dstate=None, want_dmem=False):
    BF16 = emu_ops.BF16  # (read at call time: the `exact` fixture of tests/test_autograd.py sets it to fp32)
    h = Q.shape[-1]
    D = h // heads
    T = maxlen + t
    q = Q.float().reshape(B, t, heads, D).permute(0, 2, 1, 3).requires_grad_(True)
    kf = Kf.float().requires_grad_(True)
    vf = Vf.float().requires_grad_(True)
    k = kf.reshape(B, T, heads, D).permute(0, 2, 1, 3)
    v = vf.reshape(B, T, heads, D).permute(0, 2, 1, 3)
    Rf = R.float().requires_grad_(True)
    bf = b_nd.float().requires_grad_(True)
    i = torch.arange(t)[:, None]
    j = torch.arange(T)[None, :]
    d = maxlen + i - j
    band = (d >= 0) & (d < maxlen)
    memok = torch.zeros(B, maxlen, dtype=torch.bool) if smask is None else (smask.reshape(B, maxlen) != 0)
    memok = memok & (first_u8[:, 0] == 0)[:, None]
    colok = torch.cat([memok, torch.ones(B, t, dtype=torch.bool)], 1)
    allowed = band[None] & colok[:, None, :]
    E = Rf.reshape(B, t, heads, -1).permute(0, 2, 1, 3) @ bf
    extra = torch.gather(E, 3, d.clamp(0, maxlen - 1)[None, None].expand(B, heads, t, T))
    logit = torch.where(allowed[:, None], q @ k.transpose(-1, -2) / D + extra, torch.tensor(-float("inf")))
    o = (torch.softmax(logit, -1) @ v).permute(0, 2, 1, 3).reshape(B * t, h)
    gq, gk, gv, gR, gb = torch.autograd.grad(o, [q, kf, vf, Rf, bf], dO.float().reshape(B * t, h))
    # state_out = full[t : t + maxlen]: its gradient lands on those rows of [memory | chunk], in fp32, before any rounding
    for g, ds in zip((gk, gv), (None, None) if dstate is None else dstate):
        if ds is not None:
            g[:, t:t + maxlen] += ds.float()
    out[:, 0:h] = gq.permute(0, 2, 1, 3).reshape(B * t, h).to(BF16)
    out[:, h:2 * h] = gk[:, maxlen:].reshape(B * t, h).to(BF16)
    out[:, 2 * h:3 * h] = gv[:, maxlen:].reshape(B * t, h).to(BF16)
    nr = R.shape[-1]
    out[:, 3 * h:3 * h + nr] = gR.reshape(B * t, nr).to(BF16)
    dmem = (gk[:, :maxlen].contiguous(), gv[:, :maxlen].contiguous()) if want_dmem else None
    return gb.contiguous(), dmem
