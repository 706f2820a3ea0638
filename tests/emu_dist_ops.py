"""TEST-ONLY torch emulation of the head distribution ops (video-pre-training_b200/ops_dist.py), same signatures; see emu_ops.py."""
import torch

F32 = torch.float32


def head_entropy(logp, groups=1):
    lp = logp.float()
    return -(torch.exp(lp) * lp).sum(-1)


def head_kl(logq, logp, groups=1):
    lq = logq.float()
    return (torch.exp(lq) * (lq - logp.float())).sum(-1)


def head_entropy_bwd(logp, g, groups=1):
    lp = logp.float()
    return -g.float()[:, None] * torch.exp(lp) * (lp + 1.0)


def head_kl_bwd(logq, logp, g, groups=1, want_q=True, want_p=True):
    lq = logq.float()
    gq = g.float()[:, None] * torch.exp(lq)
    return (gq * (lq - logp.float() + 1.0) if want_q else None), (-gq if want_p else None)


def rl_head_bwd_ent(logp, idx, c, logq, k, e, inv_temp, out, col0, kl=None, ent=None):
    """emu_rl_ops.rl_head_bwd plus the entropy term, added only when e != 0 (as the kernel does)."""
    rows, n = logp.shape
    lp = logp.float()
    p = torch.exp(lp)
    h = -(p * lp).sum(-1)
    g = c[:, None] * p
    g[torch.arange(rows), idx] -= c
    if logq is not None:
        q = torch.exp(logq.float())
        g = g + k * (p - q)
        r = (q * (logq.float() - lp)).sum(-1)
    else:
        r = torch.zeros(rows, dtype=F32)
    if e != 0:
        g = g + e * p * (lp + h[:, None])
    out[:, col0:col0 + n] = (g * inv_temp).to(out.dtype)
    return (r, h) if kl is None else (kl + r, ent + h)
