#!/usr/bin/env python
"""RL fine-tuning throughput: the 2x policy (the width of the released RL models) trained with RLTrainer at B = 16, T = 128 (2048 frames)
per call, on synthetic frames, actions, advantages and returns, with a frozen reference policy supplying pd_ref.  Prints the card, its
power limit and SM clock from the same run, then

  - ms per RL call (reference-policy forward excluded), frames/s and peak memory,
  - the reference-policy forward (one no-grad forward of the frozen policy on the same frames),
  - the BC step (BCTrainer) at the same shape in the same run,
  - the RL kernels' time (CUDA events around each ops.* call of one instrumented call) and their achieved bytes/s against the HBM bound
    computed from the shapes."""
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth
RL_KERNELS = ("ppo_coef", "rl_head_bwd", "ewma_sums", "value_bwd")

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=16)
ap.add_argument("--T", type=int, default=128)
ap.add_argument("--steps", type=int, default=3, help="timed calls")
ap.add_argument("--warmup", type=int, default=2)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print(f"card: {q.stdout.strip() or torch.cuda.get_device_name()}  (name, power limit, SM clock at start)")
kw = vpt_b200.policy_kwargs("2x")
torch.manual_seed(0)
pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS).cuda()
ref = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS).cuda()
ref.load_state_dict(pol.state_dict())
B, T = a.B, a.T
N = B * T
g = torch.Generator(device="cuda").manual_seed(0)
img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
with torch.no_grad():
    (pd0, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
old = pol.logprob(actions, pd0).reshape(B, T).float() + 0.1 * torch.randn(B, T, device="cuda", generator=g)
adv = torch.randn(B, T, device="cuda", generator=g)
returns = 3.0 + torch.randn(B, T, device="cuda", generator=g)
del pd0
rl, bc = vpt_b200.RLTrainer(pol), vpt_b200.BCTrainer(pol)
ref_state = ref.initial_state(B)


def ref_forward():
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref_state)
    return pd_ref


pd_ref = ref_forward()


def rl_call():
    for p in pol.parameters():
        p.grad = None
    return rl.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1)[0]


def bc_call():
    for p in pol.parameters():
        p.grad = None
    return bc.loss_and_grad(img, first, pol.initial_state(B), actions)[0]


def timed(fn):
    for _ in range(a.warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps


torch.cuda.reset_peak_memory_stats()
ms_rl = timed(rl_call)
peak = torch.cuda.max_memory_allocated() / 2 ** 30
nat.device_check()
ms_ref = timed(ref_forward)
ms_bc = timed(bc_call)
print(f"RL step, 2x policy, B={B} T={T} ({N} frames) per call: {ms_rl:.1f} ms, {N / ms_rl * 1e3:.0f} frames/s, peak memory {peak:.1f} GiB "
      f"(stats: {', '.join(f'{k} {v.item():.4f}' for k, v in rl.stats.items())})")
print(f"reference-policy forward on the same frames: {ms_ref:.1f} ms")
print(f"BC step at the same shape: {ms_bc:.1f} ms, {N / ms_bc * 1e3:.0f} frames/s")

# the RL kernels of one instrumented call (CUDA events around each ops.* call)
recs = []
orig = {n: f for n, f in vars(ops).items() if isinstance(f, types.FunctionType) and n in RL_KERNELS}


def wrap(n, f):
    def w(*args, **kwargs):
        s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0.record()
        try:
            return f(*args, **kwargs)
        finally:
            s1.record()
            recs.append((n, args[0].shape[-1] if n == "rl_head_bwd" else None, s0, s1))
    return w


for n, f in orig.items():
    setattr(ops, n, wrap(n, f))
rl_call()
torch.cuda.synchronize()
for n, f in orig.items():
    setattr(ops, n, f)
agg = collections.OrderedDict()
for n, width, s0, s1 in recs:
    v = agg.setdefault((n, width), [0, 0.0])
    v[0] += 1
    v[1] += s0.elapsed_time(s1)


def bytes_of(n, width):
    """HBM traffic the kernel needs, from the shapes (each operand read once, each result written once)."""
    if n == "rl_head_bwd":
        return N * width * (4 + 4 + 2) + N * (8 + 4 + 4 + 4)  # logp, logq fp32 in; dlog bf16 out; idx, c, kl in / out
    if n == "ppo_coef":
        return N * 4 * 6
    if n == "ewma_sums":
        return N * 4
    return N * (4 + 4 + 2 + 4)  # value_bwd: vpred, returns in; one bf16 column and the squared errors out


print("RL kernels (one call):")
tot_ms, tot_b = 0.0, 0
for (n, width), (c, t_) in agg.items():
    b = bytes_of(n, width)
    tot_ms, tot_b = tot_ms + t_, tot_b + b
    name = f"{n} (n={width})" if width else n
    print(f"  {name:24s} {t_:7.3f} ms  n={c}  {b / 1e6:7.1f} MB  {b / (t_ * 1e-3) / 1e12:5.2f} TB/s  "
          f"(HBM bound {b / HBM_BYTES_PER_S * 1e3:.3f} ms: {b / HBM_BYTES_PER_S * 1e3 / t_ * 100:.0f} % of it)")
print(f"  together {tot_ms:.3f} ms = {tot_ms / ms_rl * 100:.2f} % of the RL call; {tot_b / 1e6:.1f} MB at {tot_b / (tot_ms * 1e-3) / 1e12:.2f} TB/s")
