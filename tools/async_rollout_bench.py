#!/usr/bin/env python
"""Asynchronous rollout steps at 2x width: a graphed step of k environments picked from a ring of E, against the graphed step of a ring
of exactly k environments.

    python tools/async_rollout_bench.py [--steps 5] [--warmup 2] [--maxlens 128 1920]

For each maxlen (128, the released models; 1920, the reference's default attention_memory_size 2048) and k in {1, 8, 16, 32, 64}:
  ring_k      `GraphedAct(B=k, memory="ring")` stepping its whole ring of k environments;
  subset_E    `GraphedAct(B=k, memory="ring", envs=E)` for E = 64 and 1024, each call stepping k random distinct environments of its
              ring (`step.state.rows(idx)`; 16 such views are made before the timed runs and taken in turn, so the host-side `rows()`
              validation is not in the window);
and a padded call: 5 real rows in the B = 8 graph of envs=64 against 8 real rows.  Each number is ms per graph replay: the median over
the timed runs, each of `n` calls between two CUDA events, with the variants of one k alternating run by run.  `hbm_bound_ms` is the
bytes a step must move -- the bf16 weights plus one bf16 read of the k stepped environments' K and V memory, computed from the shapes --
over 3.35 TB/s.  A variant whose ring does not fit in memory reports null.  The card's name and power limit are read in the same run."""
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
ap.add_argument("--ks", type=int, nargs="+", default=[1, 8, 16, 32, 64])
ap.add_argument("--envs", type=int, nargs="+", default=[64, 1024])
a = ap.parse_args()
HBM = 3.35e12
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
    """A graphed ring step of B rows: of its whole ring (envs=None), or of `real` random distinct environments of a ring of `envs`."""

    def __init__(self, pol, B, envs=None, real=None, seed=0):
        g = torch.Generator().manual_seed(seed)
        real = B if real is None else real
        self.obs = {"img": torch.randint(0, 256, (real, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()}
        self.first = torch.zeros(real, dtype=torch.bool, device="cuda")
        self.act = GraphedAct(pol, B, memory="ring", envs=envs)
        if envs is None:
            self.views = [self.act.state]
        else:
            self.views = [self.act.state.rows(torch.randperm(envs, generator=g)[:real]) for _ in range(16)]
        self.i = 0

    def run(self, n):
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(n):
            self.act(self.obs, self.first, self.views[self.i % len(self.views)])
            self.i += 1
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n


def bound_ms(pol, k):
    cfg = pol.net.cfg
    w = 2 * sum(p.numel() for p in pol.parameters())
    kv = cfg.n_layers * k * 2 * cfg.maxlen * cfg.hidsize * 2
    return round((w + kv) / HBM * 1e3, 3)


def fresh():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def alternating(makers, n):
    """ms per replay of each variant, alternating run by run; None for a variant that does not fit."""
    fresh()
    rolls = {}
    for name, make in makers.items():
        try:
            rolls[name] = make()
            rolls[name].run(1)  # builds the graph
        except torch.cuda.OutOfMemoryError:
            rolls[name] = None
            fresh()
    ms = {name: [] for name in makers}
    for it in range(a.warmup + a.steps):
        for name, r in rolls.items():
            if r is not None:
                t = r.run(n)
                if it >= a.warmup:
                    ms[name].append(t)
    del rolls
    fresh()
    return {name: (round(median(v), 3) if v else None) for name, v in ms.items()}


def main():
    name, power = card()
    res = dict(card=name, power_limit=power, hbm_tb_s=HBM / 1e12)
    for maxlen in a.maxlens:
        pol = policy(maxlen)
        out = {}
        for k in a.ks:
            n = 20 if k <= 16 else 10
            makers = {"ring_k": lambda k=k: Roll(pol, k, seed=k)}
            for E in a.envs:
                makers[f"subset_{E}"] = lambda k=k, E=E: Roll(pol, k, envs=E, seed=k)
            out[f"k{k}"] = dict(alternating(makers, n), hbm_bound_ms=bound_ms(pol, k))
            print(json.dumps({f"maxlen{maxlen}": {f"k{k}": out[f"k{k}"]}}), flush=True)
        out["padded"] = dict(alternating({"B8_8rows": lambda: Roll(pol, 8, envs=64, seed=8),
                                          "B8_5rows": lambda: Roll(pol, 8, envs=64, real=5, seed=5)}, 20),
                             hbm_bound_ms_8rows=bound_ms(pol, 8), hbm_bound_ms_5rows=bound_ms(pol, 5))
        print(json.dumps({f"maxlen{maxlen}": {"padded": out["padded"]}}), flush=True)
        res[f"maxlen{maxlen}"] = out
        del pol
        fresh()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
