"""TEST-ONLY torch emulation of the RL fine-tuning ops (video-pre-training_b200/ops_rl.py), same signatures; see emu_ops.py."""
import torch

F32 = torch.float32


def ppo_coef(lp, old_logprob, advantages, clip):
    rows = lp.numel()
    lo, hi = torch.tensor(1.0 - clip, dtype=F32), torch.tensor(1.0 + clip, dtype=F32)
    ratio = torch.exp(lp.float() - old_logprob.float())
    a = advantages.float()
    clipped = ((a > 0) & (ratio > hi)) | ((a < 0) & (ratio < lo))
    surr1, surr2 = ratio * a, torch.minimum(torch.maximum(ratio, lo), hi) * a
    c = torch.where(clipped, torch.zeros_like(ratio), surr1 / rows)
    return c, -torch.minimum(surr1, surr2), clipped.float()


def rl_head_bwd(logp, idx, c, logq, k, inv_temp, out, col0, kl=None):
    rows, n = logp.shape
    p = torch.exp(logp.float())
    g = c[:, None] * p
    g[torch.arange(rows), idx] -= c
    if logq is not None:
        q = torch.exp(logq.float())
        g = g + k * (p - q)
        r = (q * (logq.float() - logp.float())).sum(-1)
    else:
        r = torch.zeros(rows, dtype=F32)
    out[:, col0:col0 + n] = (g * inv_temp).to(out.dtype)
    return r if kl is None else kl + r


def ewma_sums(x):
    x = x.double()
    return torch.stack([x.sum(), (x * x).sum()])


def value_bwd(vpred, returns, sums, count, running_mean, running_mean_sq, debiasing_term, beta, scale, out, col):
    """lib/normalize_ewma.py:36-55 in training mode (the update in the reference's fp32 operation order), then the scaled MSE gradient."""
    with torch.no_grad():
        bm, bsq = (sums / count).float()
        running_mean.mul_(beta).add_(bm * (1.0 - beta))
        running_mean_sq.mul_(beta).add_(bsq * (1.0 - beta))
        debiasing_term.mul_(beta).add_(1.0 * (1.0 - beta))
        deb = debiasing_term.clamp(min=1e-5)
        mean = running_mean / deb
        var = (running_mean_sq / deb - mean ** 2).clamp(min=1e-2)
        d = vpred.reshape(-1).float() - (returns.reshape(-1).float() - mean) / torch.sqrt(var)
        out[:, col] = (scale * d).to(out.dtype)
    return d * d
