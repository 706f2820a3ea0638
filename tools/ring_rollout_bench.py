#!/usr/bin/env python
"""Rollout steps at 2x width with the KV memory as the reference's pytree against the in-place ring (`RingState`):
`GraphedAct(memory="pytree")` against `GraphedAct(memory="ring")` at maxlen 128 (the released models) and 1920 (the reference's default
attention_memory_size 2048), for B = 1, B = 64 and the largest B that fits each way.

    python tools/ring_rollout_bench.py [--steps 5] [--warmup 2]

For each (maxlen, B, memory): ms per step (median over the timed runs of `n` graph replays, CUDA events; at B = 1 and 64 the two
memories alternate run by run), the peak memory of the process, and the bytes a step must move -- the bf16 weights plus one bf16 read of
every layer's K and V memory, computed from the shapes -- against the HBM bound (3.35 TB/s).  The largest B is found from the peak memory
at B = 16 and 32 (its per-environment slope), then stepped down by 10% until a GraphedAct of that size builds and runs.  The card's name
and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200.policy import GraphedAct

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--maxlens", type=int, nargs="+", default=[128, 1920])
a = ap.parse_args()
HBM = 3.35e12
MEMORIES = ("pytree", "ring")
ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731


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


def policy(maxlen):
    torch.manual_seed(0)
    kw = vpt_b200.policy_kwargs("2x", attention_memory_size=maxlen + 128)
    return vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS).cuda()


class Roll:
    """A GraphedAct of one memory kind and batch size, its inputs and its state."""

    def __init__(self, pol, B, memory):
        g = torch.Generator(device="cuda").manual_seed(B)
        self.obs = {"img": torch.randint(0, 256, (B, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)}
        self.first = torch.zeros(B, dtype=torch.bool, device="cuda")
        self.act = GraphedAct(pol, B, memory=memory)
        self.state = self.act.state

    def run(self, n):
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(n):
            _, self.state, _ = self.act(self.obs, self.first, self.state)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n


def step_bytes(pol, B):
    cfg = pol.net.cfg
    w = 2 * sum(p.numel() for p in pol.parameters())
    kv = cfg.n_layers * B * 2 * cfg.maxlen * cfg.hidsize * 2
    return w, kv


def report(pol, B, ms, peak):
    w, kv = step_bytes(pol, B)
    return dict(B=B, ms=round(ms, 3), peak_gib=round(peak, 2), step_mb=round((w + kv) / 1e6, 1), hbm_bound_ms=round((w + kv) / HBM * 1e3, 3))


def fresh():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def alternating(pol, B, n):
    """Both memories at one B, alternating run by run; the peak memory of each on its own."""
    peaks = {m: peak_of(pol, B, m) / 2**30 for m in MEMORIES}
    fresh()
    rolls = {m: Roll(pol, B, m) for m in MEMORIES}
    ms = {m: [] for m in MEMORIES}
    for it in range(a.warmup + a.steps):
        for m in MEMORIES:
            t = rolls[m].run(n)
            if it >= a.warmup:
                ms[m].append(t)
    del rolls
    return {m: report(pol, B, median(ms[m]), peaks[m]) for m in MEMORIES}


def peak_of(pol, B, memory):
    fresh()
    r = Roll(pol, B, memory)
    r.run(2)
    p = torch.cuda.max_memory_allocated()
    del r
    return p


def largest(pol, memory, n):
    """The largest B (a multiple of 8) whose GraphedAct builds and runs, from the peak memory's slope over B."""
    p16, p32 = peak_of(pol, 16, memory), peak_of(pol, 32, memory)
    slope = (p32 - p16) / 16
    total = torch.cuda.get_device_properties(0).total_memory
    B = int((0.92 * total - (p16 - 16 * slope)) / slope) // 8 * 8
    for _ in range(6):
        try:
            fresh()
            r = Roll(pol, B, memory)
            ms = [r.run(n) for _ in range(a.warmup + a.steps)][a.warmup:]
            peak = torch.cuda.max_memory_allocated() / 2**30
            del r
            return dict(report(pol, B, median(ms), peak), per_env_mb=round(slope / 1e6, 2))
        except torch.cuda.OutOfMemoryError:
            r = None
            B = int(B * 0.9) // 8 * 8
    return dict(B=None, per_env_mb=round(slope / 1e6, 2))


def main():
    name, power = card()
    res = dict(card=name, power_limit=power, hbm_tb_s=HBM / 1e12)
    for maxlen in a.maxlens:
        pol = policy(maxlen)
        out = {}
        for B, n in ((1, 20), (64, 10)):
            out[f"B{B}"] = alternating(pol, B, n)
        out["largest"] = {m: largest(pol, m, 3) for m in MEMORIES}
        res[f"maxlen{maxlen}"] = out
        print(json.dumps({f"maxlen{maxlen}": out}), flush=True)
        del pol
        fresh()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
