"""Tensor-level wrapper of the attention backward with gradients through the KV memory (csrc/attention_bwd.cuh, `vpt_attention_bwd_state`),
re-exported by `ops`; same conventions as ops.py.  It backs the differentiable forward's `state_grad` (truncated BPTT across calls)."""
import torch

from . import _native as nat
from . import ops

F32 = torch.float32


def attention_bwd_state(Q, Kf, Vf, R, b_nd, first_u8, smask, dO, out, B, t, maxlen, heads, dstate=None, want_dmem=False):
    """`ops.attention_bwd` (causal) with the KV memory in the graph.  state_out = rows t .. t+maxlen of [memory|chunk].
    dstate: None or a pair (dk, dv), either None, of fp32 contiguous (B, maxlen, h): the upstream gradient wrt this call's state_out K / V,
    added in fp32 to the chunk rows it came from before their bf16 rounding (and, with t < maxlen, passed through to the memory rows).
    want_dmem: also compute the gradient wrt state_in K / V.
    Writes d q | d k | d v | d R into `out` like `attention_bwd` and returns (d b_nd, (dmem_k, dmem_v) fp32 (B, maxlen, h) or None)."""
    ops._cuda(Q, Kf, Vf, R, b_nd, dO, out)
    h = heads * 128
    ds = (None, None) if dstate is None else tuple(dstate)
    if len(ds) != 2:
        raise ValueError("attention_bwd_state: dstate must be a pair (dk, dv)")
    shape = (B, maxlen, h)
    for name, x in zip(("dstate[0]", "dstate[1]"), ds):
        if x is None:
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != F32 or tuple(x.shape) != shape or not x.is_contiguous() or x.data_ptr() % 16:
            raise ValueError(f"attention_bwd_state: {name} must be a contiguous 16-byte aligned fp32 tensor of shape {shape} "
                             f"(got {getattr(x, 'dtype', type(x).__name__)} {tuple(getattr(x, 'shape', ()))})")
        ops._cuda(x)
    nbasis = b_nd.shape[0]
    ws = torch.empty((2, B * heads, t, maxlen), dtype=F32, device=Q.device)  # P and dS by relative distance d
    db = torch.empty((nbasis, maxlen), dtype=F32, device=Q.device)
    dmem = (torch.empty(shape, dtype=F32, device=Q.device), torch.empty(shape, dtype=F32, device=Q.device)) if want_dmem else (None, None)
    nat.check(nat.lib().vpt_attention_bwd_state(ops._p(Q), ops._p(Kf), ops._p(Vf), ops._p(R), R.stride(-2), ops._p(b_nd), ops._p(first_u8),
                                                first_u8.stride(0), ops._p(smask), ops._p(dO), ops._p(out), out.stride(0), ops._p(db),
                                                ops._p(ws), B, t, maxlen, heads, nbasis, ops._p(ds[0]), ops._p(ds[1]), ops._p(dmem[0]),
                                                ops._p(dmem[1]), ops._stream()), "vpt_attention_bwd_state")
    ops._count(4 if want_dmem else 3)
    return db, (dmem if want_dmem else None)
