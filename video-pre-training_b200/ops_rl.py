"""Tensor-level wrappers of the RL fine-tuning kernels (csrc/rl_bwd.cuh), re-exported by `ops`; same conventions as ops.py."""
import torch

from . import _native as nat
from . import ops

F32 = torch.float32


def _rows_f32(name, what, t, rows):
    if t.dtype != F32 or t.numel() != rows or not t.is_contiguous():
        raise ValueError(f"{name}: {what} must be contiguous fp32 with {rows} elements (got {t.dtype} {tuple(t.shape)})")


def ppo_coef(lp, old_logprob, advantages, clip):
    """Per-row PPO coefficient of the policy-gradient term: lp, old_logprob, advantages fp32 [rows] ->
    (c, pi_loss, clipped) fp32 [rows]: c = ratio * A / rows, 0 where the objective is clipped; the row's clipped surrogate loss; 1 / 0."""
    ops._cuda(lp, old_logprob, advantages)
    rows = lp.numel()
    for what, t in (("lp", lp), ("old_logprob", old_logprob), ("advantages", advantages)):
        _rows_f32("ppo_coef", what, t, rows)
    if not 0.0 <= clip < 1.0:
        raise ValueError(f"ppo_coef: clip must lie in [0, 1) (got {clip})")
    c, pi_loss, clipped = (torch.empty((rows,), dtype=F32, device=lp.device) for _ in range(3))
    nat.check(nat.lib().vpt_ppo_coef(ops._p(lp), ops._p(old_logprob), ops._p(advantages), rows, 1.0 - clip, 1.0 + clip, 1.0 / rows, ops._p(c),
                                     ops._p(pi_loss), ops._p(clipped), ops._stream()), "vpt_ppo_coef")
    ops._count()
    return c, pi_loss, clipped


def rl_head_bwd(logp, idx, c, logq, k, inv_temp, out, col0, kl=None):
    """One categorical head: logp fp32 [rows, n] (and logq, the frozen reference policy's, or None), idx int64 [rows] ->
    out[:, col0:col0+n] = (c[r] * (exp(logp) - onehot(idx)) + k * (exp(logp) - exp(logq))) * inv_temp (bf16); returns kl fp32 [rows] =
    KL(exp(logq) || exp(logp)) per row (added to `kl` when given; zeros without logq)."""
    ops._cuda(logp, idx, c, logq, out, kl)
    if logp.dtype != F32 or logp.dim() != 2 or logp.stride(1) != 1:
        raise ValueError("rl_head_bwd: logp must be fp32 [rows, n] with unit column stride")
    rows, n = logp.shape
    if logq is not None and (logq.dtype != F32 or tuple(logq.shape) != (rows, n) or logq.stride(1) != 1):
        raise ValueError(f"rl_head_bwd: logq must be fp32 [{rows}, {n}] with unit column stride")
    if idx.dtype != torch.int64 or idx.numel() != rows or not idx.is_contiguous():
        raise ValueError(f"rl_head_bwd: idx must be contiguous int64 with {rows} elements")
    _rows_f32("rl_head_bwd", "c", c, rows)
    if out.dtype != torch.bfloat16 or out.dim() != 2 or out.shape[0] != rows or out.shape[1] < col0 + n or col0 < 0 or out.stride(1) != 1:
        raise ValueError("rl_head_bwd: out must be bf16 [rows, >= col0 + n] with unit column stride")
    if rows and (int(idx.min()) < 0 or int(idx.max()) >= n):  # (one host sync: the kernel would index past the head's columns)
        raise ValueError(f"rl_head_bwd: actions must lie in [0, {n})")
    acc = kl is not None
    if kl is None:
        kl = torch.empty((rows,), dtype=F32, device=logp.device)
    else:
        _rows_f32("rl_head_bwd", "kl", kl, rows)
    nat.check(nat.lib().vpt_rl_head_bwd(ops._p(logp), logp.stride(0), ops._p(logq), 0 if logq is None else logq.stride(0), ops._p(idx), ops._p(c),
                                        float(k), float(inv_temp), n, ops._p(out), out.stride(0), col0, ops._p(kl), int(acc), rows, ops._stream()),
              "vpt_rl_head_bwd")
    ops._count()
    return kl


def ewma_sums(x):
    """float64 [2] = (sum, sum of squares) of the fp32 values x."""
    ops._cuda(x)
    _rows_f32("ewma_sums", "x", x, x.numel())
    if x.numel() == 0:
        raise ValueError("ewma_sums: x is empty")
    sums = torch.empty((2,), dtype=torch.float64, device=x.device)
    nat.check(nat.lib().vpt_ewma_sums(ops._p(x), x.numel(), ops._p(sums), ops._stream()), "vpt_ewma_sums")
    ops._count()
    return sums


def value_bwd(vpred, returns, sums, count, running_mean, running_mean_sq, debiasing_term, beta, scale, out, col):
    """Value head in training mode: updates the EWMA normaliser (running_mean, running_mean_sq, debiasing_term: fp32, one element each) in
    place with the batch statistics sums / count (sums from `ewma_sums`, all-reduced under data parallelism), then writes
    scale * (vpred - normalised returns) (bf16) into out[:, col]; returns the squared errors fp32 [rows]."""
    ops._cuda(vpred, returns, sums, running_mean, running_mean_sq, debiasing_term, out)
    rows = vpred.numel()
    _rows_f32("value_bwd", "vpred", vpred, rows)
    _rows_f32("value_bwd", "returns", returns, rows)
    for what, t in (("running_mean", running_mean), ("running_mean_sq", running_mean_sq), ("debiasing_term", debiasing_term)):
        _rows_f32("value_bwd", what, t, 1)
    if sums.dtype != torch.float64 or tuple(sums.shape) != (2,) or not sums.is_contiguous():
        raise ValueError("value_bwd: sums must be contiguous float64 [2]")
    if out.dtype != torch.bfloat16 or out.dim() != 2 or out.shape[0] != rows or not 0 <= col < out.shape[1] or out.stride(1) != 1:
        raise ValueError(f"value_bwd: out must be bf16 [{rows}, > col] with unit column stride")
    if count <= 0:
        raise ValueError("value_bwd: count must be positive")
    sq = torch.empty((rows,), dtype=F32, device=vpred.device)
    nat.check(nat.lib().vpt_value_bwd(ops._p(vpred), ops._p(returns), ops._p(sums), float(count), ops._p(running_mean), ops._p(running_mean_sq),
                                      ops._p(debiasing_term), float(beta), 1.0 - float(beta), float(scale), ops._p(out), out.stride(0), col,
                                      ops._p(sq), rows, ops._stream()), "vpt_value_bwd")
    ops._count()
    for t in (running_mean, running_mean_sq, debiasing_term):  # written behind autograd's back: let version-keyed caches see the change
        torch.autograd.graph.increment_version(t)
    return sq
