"""TEST INFRASTRUCTURE: float64 references for `vpt_attention_bwd_state` (the attention backward with the KV memory in the graph).

`closed_form` writes the backward out (P, dS, then dK / dV over every row of [memory | chunk]) the way the kernel computes it;
`by_autograd` is torch autograd of the attention (the formulas of tests/bwd_refs.py, from the oracle) with the memory rows as leaves and
the state_out gradient entering through a linear term.  tests/test_bptt.py checks the first against the second on the CPU;
tests/test_gpu_bptt.py checks the kernel against the first."""
import torch

import vpt_oracle as O

F64 = torch.float64


def _setup(first_u8, smask_u8, B, t, maxlen, dev):
    T = maxlen + t
    smask = None if smask_u8 is None else (smask_u8.reshape(B, 1, maxlen) != 0)
    with torch.device(dev):
        mask, _ = O.allowed_mask(first_u8[:, 0] != 0, smask, t, maxlen)
        d = (T - t + torch.arange(t)[:, None]) - torch.arange(T)[None, :]
    return mask, d, (d >= 0) & (d < maxlen)


def closed_form(Q, Kf, Vf, R, b_nd, first_u8, smask_u8, dO, B, t, maxlen, heads, dstate=(None, None)):
    """-> dict(dq, dk, dv [B*t][h] (chunk rows), dR, db_nd, dmem_k, dmem_v (B, maxlen, h)), float64."""
    dev = Q.device
    h = Q.shape[-1]
    D = h // heads
    T = maxlen + t
    mask, d, okb = _setup(first_u8, smask_u8, B, t, maxlen, dev)
    q = Q.to(F64).reshape(B, t, heads, D).permute(0, 2, 1, 3)
    k = Kf.to(F64).reshape(B, T, heads, D).permute(0, 2, 1, 3)
    v = Vf.to(F64).reshape(B, T, heads, D).permute(0, 2, 1, 3)
    Rh = R.to(F64).reshape(B, t, heads, -1).permute(0, 2, 1, 3)                        # (B, heads, t, nbasis)
    Dm = torch.where(okb[None], b_nd.to(F64)[:, d.clamp(0, maxlen - 1)], torch.zeros((), dtype=F64, device=dev))  # (nbasis, t, T)
    extra = torch.einsum("bhin,nij->bhij", Rh, Dm)
    S = q @ k.transpose(-1, -2) / D + extra
    S = S.masked_fill(~mask[:, None], -float("inf"))
    P = torch.softmax(S, -1)
    g = dO.to(F64).reshape(B, t, heads, D).permute(0, 2, 1, 3)
    dP = g @ v.transpose(-1, -2)
    dS = P * (dP - (P * dP).sum(-1, keepdim=True))
    dq = dS @ k / D
    dk = dS.transpose(-1, -2) @ q / D                                                     # (B, heads, T, D): every row of [memory | chunk]
    dv = P.transpose(-1, -2) @ g
    dR = torch.einsum("bhij,nij->bhin", dS, Dm)
    dbf = torch.einsum("bhij,bhin->nij", dS, Rh)
    db = torch.zeros(b_nd.shape, dtype=F64, device=dev)
    for dd in range(maxlen):
        db[:, dd] = (dbf * (d == dd)[None]).sum((1, 2))
    merge = lambda x: x.permute(0, 2, 1, 3).reshape(B, -1, h)  # noqa: E731
    dk, dv = merge(dk), merge(dv)
    for full, ds in zip((dk, dv), dstate):
        if ds is not None:
            full[:, t:t + maxlen] += ds.to(F64)
    return dict(dq=merge(dq).reshape(B * t, h), dk=dk[:, maxlen:].reshape(B * t, h), dv=dv[:, maxlen:].reshape(B * t, h),
                dR=dR.permute(0, 2, 1, 3).reshape(B * t, -1), db_nd=db, dmem_k=dk[:, :maxlen], dmem_v=dv[:, :maxlen])


def by_autograd(Q, Kf, Vf, R, b_nd, first_u8, smask_u8, dO, B, t, maxlen, heads, dstate=(None, None)):
    """The same gradients by torch autograd, float64: the memory rows are leaves, and state_out = full[:, t:t+maxlen] meets dstate."""
    dev = Q.device
    h = Q.shape[-1]
    T = maxlen + t
    q = Q.to(F64).clone().requires_grad_(True)
    fk = Kf.to(F64).clone().requires_grad_(True)
    fv = Vf.to(F64).clone().requires_grad_(True)
    Rr = R.to(F64).clone().requires_grad_(True)
    bn = b_nd.to(F64).clone().requires_grad_(True)
    mask, d, okb = _setup(first_u8, smask_u8, B, t, maxlen, dev)
    Dm = torch.where(okb[None], bn[:, d.clamp(0, maxlen - 1)], torch.zeros((), dtype=F64, device=dev))
    Qh, Kh, Vh = O.split_heads(q.reshape(B, t, h), heads), O.split_heads(fk, heads), O.split_heads(fv, heads)
    Rh = O.split_heads(Rr.reshape(B, t, -1), heads)
    e = Qh.shape[2]
    bias = (~mask).to(F64).repeat_interleave(heads, dim=0) * -1e9 + torch.einsum("btn,ntp->btp", Rh, Dm)
    Wt = torch.softmax(torch.baddbmm(bias, Qh, Kh.transpose(-1, -2), alpha=1.0 / e), dim=2)
    A = torch.einsum("btp,bpe->bte", Wt, Vh).reshape(B, heads, t, e).permute(0, 2, 1, 3).reshape(B * t, h)
    loss = (A * dO.to(F64)).sum()
    for full, ds in zip((fk, fv), dstate):
        if ds is not None:
            loss = loss + (full[:, t:t + maxlen] * ds.to(F64)).sum()
    dq, dk, dv, dR, db = torch.autograd.grad(loss, (q, fk, fv, Rr, bn))
    return dict(dq=dq, dk=dk[:, maxlen:].reshape(B * t, h), dv=dv[:, maxlen:].reshape(B * t, h), dR=dR, db_nd=db, dmem_k=dk[:, :maxlen],
                dmem_v=dv[:, :maxlen])


def inputs(B, t, maxlen, heads, seed, dev="cpu", with_dstate=True):
    """Seeded kernel inputs: bf16-valued Q / K / V / dO, fp32 R (10 basis rows per head) and b_nd, `first` resets on every third batch row
    and a partial state_mask; dstate fp32 (B, maxlen, h) pair or (None, None)."""
    g = torch.Generator().manual_seed(seed)
    h = heads * 128
    T = maxlen + t
    bf = lambda *s: (torch.randn(*s, generator=g) * 2.0).to(torch.bfloat16)  # noqa: E731
    Q, Kf, Vf, dO = bf(B * t, h), bf(B, T, h), bf(B, T, h), (torch.randn(B * t, h, generator=g) * 0.1).to(torch.bfloat16)
    R = torch.randn(B * t, 10 * heads, generator=g)
    b_nd = torch.randn(10, maxlen, generator=g)
    first = torch.zeros(B, t, dtype=torch.bool)
    first[::3, 0] = True
    smask = torch.rand(B, maxlen, generator=g) > 0.25
    ds = (torch.randn(B, maxlen, h, generator=g) * 0.05, torch.randn(B, maxlen, h, generator=g) * 0.05) if with_dstate else (None, None)
    to = lambda x: None if x is None else x.to(dev)  # noqa: E731
    return dict(Q=to(Q), Kf=to(Kf), Vf=to(Vf), R=to(R), b_nd=to(b_nd), first_u8=to(first.view(torch.uint8)), smask_u8=to(smask.view(torch.uint8)),
                dO=to(dO), dstate=tuple(to(x) for x in ds))
