#!/usr/bin/env python
"""What the batch-invariant mode costs (`MinecraftAgentPolicy.set_batch_invariant`), at 2x width.

    python tools/invariant_rollout_bench.py [--runs 5] [--maxlens 128 1920] [--out FILE]

Rollout steps: `GraphedAct` ms per step, default mode against the batch-invariant mode, for maxlen 128 (the released models) and 1920:
  B = 1, 8 and 64 stepping a view of B environments of a ring of 64 (`GraphedAct(B, memory="ring", envs=64)`);
  the largest B that fits, a whole-ring `GraphedAct(B, memory="ring")` (tried from the largest ring batch that fits in the default mode,
  halved until the invariant graph fits too).
GEMM: the weight-streaming kernel at any M (`ops.gemm_rowwise`) against the default kernel choice at the same M, on the 2x model's
mlp0 shape (N = 8192, K = 2048), M = 1, 9, 64 and 1024.  `hbm_bound_ms` is the bytes the product must move at least -- the bf16 weights
once, the input rows and the output rows -- over 3.35 TB/s.
Each number is the median over the runs of device-event time per call, the two variants alternating run by run.  The card's name and
power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import ops
from video_pre_training_b200.policy import GraphedAct

ap = argparse.ArgumentParser()
ap.add_argument("--runs", type=int, default=5)
ap.add_argument("--maxlens", type=int, nargs="+", default=[128, 1920])
ap.add_argument("--largest", type=int, nargs="+", default=[8184, 1096], help="the default mode's largest ring batch, per maxlen")
ap.add_argument("--out", default=None)
a = ap.parse_args()
HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, n):
    """{name: median ms per call}, the variants alternating run by run (each warmed up first)."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(a.runs):
        for k, f in fns.items():
            t[k].append(timed(f, n))
    return {k: round(median(v), 4) for k, v in t.items()}


def step_fn(pol, ga, inv, obs, first, state):
    def f():
        pol.set_batch_invariant(inv, seed=1)
        ga(obs, first, state)
    return f


def rollout(maxlen, largest):
    torch.manual_seed(0)
    kw = vpt_b200.policy_kwargs("2x", attention_memory_size=maxlen + 128)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS).cuda()
    H = pol.net.cfg.img_shape[0]
    rows = []
    for B in (1, 8, 64):
        ga = GraphedAct(pol, B, memory="ring", envs=64)
        obs = {"img": torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device="cuda")}
        first = torch.zeros(B, dtype=torch.bool, device="cuda")
        view = ga.state.rows(torch.randperm(64)[:B])
        t = alternate({m: step_fn(pol, ga, m == "invariant", obs, first, view) for m in ("default", "invariant")}, 20 if B < 64 else 5)
        rows.append(dict(maxlen=maxlen, B=B, ring=64, **{f"{k}_ms": v for k, v in t.items()}))
        del ga
        torch.cuda.empty_cache()
    B = largest
    while B >= 64:
        ga = None
        try:
            ga = GraphedAct(pol, B, memory="ring")
            obs = {"img": torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device="cuda")}
            first = torch.zeros(B, dtype=torch.bool, device="cuda")
            t = alternate({m: step_fn(pol, ga, m == "invariant", obs, first, ga.state) for m in ("default", "invariant")}, 2)
            rows.append(dict(maxlen=maxlen, B=B, ring=B, **{f"{k}_ms": v for k, v in t.items()}))
            break
        except torch.cuda.OutOfMemoryError:
            del ga
            torch.cuda.empty_cache()
            B //= 2
    pol.set_batch_invariant(False)
    del pol
    torch.cuda.empty_cache()
    return rows


def gemm_rows():
    N, K = 8192, 2048
    W = torch.randn(N, K, device="cuda").bfloat16()
    S2 = torch.randn(N, device="cuda")
    out = []
    for M in (1, 9, 64, 1024):
        A = torch.randn(M, K, device="cuda").bfloat16()
        o = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        t = alternate({"default": lambda: ops.gemm(A, W, o, M, N, K, S2=S2, relu=1),
                       "rowwise": lambda: ops.gemm_rowwise(A, W, o, M, N, K, S2=S2, relu=1)}, 50 if M < 1024 else 10)
        bound = (N * K + M * K + M * N) * 2 / HBM * 1e3
        out.append(dict(M=M, N=N, K=K, default_ms=t["default"], rowwise_ms=t["rowwise"], hbm_bound_ms=round(bound, 4),
                        weight_streams=(M + 7) // 8))
    return out


name, power = card()
res = dict(card=name, power_limit=power, gemm=gemm_rows(), rollout=[])
for maxlen, largest in zip(a.maxlens, a.largest):
    res["rollout"] += rollout(maxlen, largest)
line = json.dumps(res)
print(line)
if a.out:
    with open(a.out, "w") as f:
        f.write(line + "\n")
