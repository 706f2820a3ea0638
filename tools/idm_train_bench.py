#!/usr/bin/env python
"""IDM training throughput: the 4x IDM (idm_net_kwargs()) trained with IDMTrainer at B = 4, T = 128 (512 frames) per call and
`--accum` calls per FlatAdamDP.step, on synthetic frames and actions.  Prints the card, its power limit and SM clock from the same
run, ms per 512-frame call, frames/s, the achieved whole-step TFLOP/s over 3 x the forward's algorithmic FLOPs, peak memory, and the
per-op breakdown of one call (CUDA events around every ops.* call, as tools/idm_bench.py) with the IDM backward kernels on their own
lines (the conv3d backward against its HBM bound)."""
import argparse
import collections
import os
import subprocess
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth

ap = argparse.ArgumentParser()
ap.add_argument("--accum", type=int, default=2, help="calls per optimizer step")
ap.add_argument("--steps", type=int, default=3, help="timed optimizer steps")
ap.add_argument("--warmup", type=int, default=2)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print(f"card: {q.stdout.strip() or torch.cuda.get_device_name()}  (name, power limit, SM clock at start)")
kw = vpt_b200.idm_net_kwargs()
torch.manual_seed(0)
pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), kw).cuda()
cfg = pol.net.cfg
tr = vpt_b200.IDMTrainer(pol)
opt = FlatAdamDP(vpt_b200.IDMTrainer.optimizer_params(pol), lr=1e-5)  # every parameter but lastlayer.*, conv3d_layer.* first
B, T = 4, 128
g = torch.Generator(device="cuda").manual_seed(0)
batches = [(torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g),
            {"buttons": torch.randint(0, 2, (B, T, 20), device="cuda", generator=g), "camera": torch.randint(0, 11, (B, T, 2), device="cuda", generator=g)})
           for _ in range(a.accum)]
first = torch.zeros(B, T, dtype=torch.bool, device="cuda")


def step():
    opt.zero_grad()
    loss = None
    for img, act in batches:
        loss, _ = tr.loss_and_grad(img, first, pol.initial_state(B), act)
    opt.step()
    return loss


for _ in range(a.warmup):
    step()
torch.cuda.synchronize()
nat.device_check()
torch.cuda.reset_peak_memory_stats()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(a.steps):
    loss = step()
e1.record()
torch.cuda.synchronize()
ms_step = e0.elapsed_time(e1) / a.steps
ms_call = ms_step / a.accum
frames = B * T
tflops = 3 * cfg.forward_flops_per_frame(head_outputs=40 + 22) * frames / (ms_call * 1e-3) / 1e12
print(f"IDM 4x training, B={B} T={T} per call, {a.accum} calls per Adam step: {ms_step:.1f} ms/step, {ms_call:.1f} ms per {frames}-frame call, "
      f"{frames / ms_call * 1e3:.0f} frames/s, loss {loss.item():.4f}")
print(f"whole-step rate over 3 x forward FLOPs: {tflops:.0f} TFLOP/s; peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")

# per-op breakdown of one call (nested ops count in the outer one)
recs, depth = [], [0]
orig = {n: f for n, f in vars(ops).items() if isinstance(f, types.FunctionType) and not n.startswith("_")}


def wrap(n, f):
    def w(*args, **kwargs):
        if depth[0]:
            return f(*args, **kwargs)
        depth[0] += 1
        s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0.record()
        try:
            return f(*args, **kwargs)
        finally:
            s1.record()
            depth[0] -= 1
            recs.append(("attention_bwd (causal=False)" if n == "attention_bwd" and kwargs.get("causal", True) is False else n, s0, s1))
    return w


for n, f in orig.items():
    setattr(ops, n, wrap(n, f))
opt.zero_grad()
e0.record()
tr.loss_and_grad(batches[0][0], first, pol.initial_state(B), batches[0][1])
e1.record()
torch.cuda.synchronize()
for n, f in orig.items():
    setattr(ops, n, f)
agg = collections.OrderedDict()
for n, s0, s1 in recs:  # (only names and events are kept: holding the arguments would keep the whole tape alive)
    v = agg.setdefault(n, [0, 0.0])
    v[0] += 1
    v[1] += s0.elapsed_time(s1)
call_ms = e0.elapsed_time(e1)
print(f"instrumented call {call_ms:.1f} ms; sum of ops {sum(v[1] for v in agg.values()):.1f} ms")
for n, (c, t_) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:16]:
    print(f"  {t_:8.2f} ms  n={c:4d}  {n}")
new = {k: agg.get(k, [0, 0.0]) for k in ("conv3d_t5_bwd", "attention_bwd (causal=False)", "softmax_nll_bwd_grouped")}
H, W, C3 = cfg.img_shape[0], cfg.img_shape[1], cfg.conv3d_out
c3_bytes = frames * ((H + 1) * (W + 1) * C3 * 2 + H * W * 3)  # bf16 dy + u8 frames
print("IDM backward kernels:")
for k, (c, t_) in new.items():
    extra = ""
    if k == "conv3d_t5_bwd" and t_ > 0:
        bound = c3_bytes / HBM_BYTES_PER_S * 1e3
        extra = f"  (reads {c3_bytes / 1e9:.2f} GB: HBM bound {bound:.2f} ms at {HBM_BYTES_PER_S / 1e12:.2f} TB/s, {bound / t_ * 100:.0f} % of it)"
    print(f"  {k:30s} {t_:7.3f} ms  n={c}{extra}")
share = sum(v[1] for v in new.values()) / call_ms * 100
print(f"  together {sum(v[1] for v in new.values()):.2f} ms = {share:.2f} % of the instrumented call")
