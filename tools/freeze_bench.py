#!/usr/bin/env python
"""Training part of the policy (`requires_grad_(False)`) against training all of it: ms per training step, peak memory and kernel launches.

    python tools/freeze_bench.py [--steps 3] [--warmup 1] [--only bc2x,big2x,rl2x]

    bc2x    2x BC at B = 16, T = 128 (BCTrainer + FlatAdamDP.step over the trainable parameters): all trainable, the CNN
            (`img_process.cnn.*`) frozen, everything below the transformer (`img_process.*`) frozen, only the heads training
    big2x   2x BC at B = 128, T = 128 in one call: the CNN frozen without recompute_frames, against all trainable with recompute_frames = 2048
    rl2x    the 2x RL step at B = 16, T = 128 (RLTrainer + FlatAdamDP.step): all trainable against the CNN frozen

Times are CUDA events around the whole step (medians over the timed steps, the variants alternating), peak memory is
`max_memory_allocated` reset before each timed step, launches are `ops.LAUNCHES` per step.  Every variant has its own policy (the same
seed) and its own FlatAdamDP over its trainable parameters.  The card's name and power limit are read in the same run."""
import argparse
import gc
import os
import subprocess
import sys

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--only", default="bc2x,big2x,rl2x")
a = ap.parse_args()
T = 128
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


def frames(g, B):
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
               "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
    return img, torch.zeros(B, T, dtype=torch.bool, device="cuda"), actions


def policy(frozen=(), keep=None, value_head=False):
    """The 2x policy with the parameters under `frozen` (or, with `keep`, all but those under `keep`) frozen, and its optimizer."""
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
    for n, p in pol.named_parameters():
        if n.startswith(tuple(frozen)) or (keep is not None and not n.startswith(keep)):
            p.requires_grad_(False)
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if value_head or not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)
    return pol, opt


def timed(variants):
    """variants: {label: step function}; warm-up, then alternating timed rounds; prints median ms, peak GiB and launches per step."""
    for _ in range(a.warmup):
        for fn in variants.values():
            fn()
    torch.cuda.synchronize()
    nat.device_check()
    times, peaks, launches = ({k: [] for k in variants} for _ in range(3))
    for _ in range(a.steps):
        for k, fn in variants.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            n0 = ops.LAUNCHES
            e0, e1 = ev(), ev()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            peaks[k].append(torch.cuda.max_memory_allocated() / 2 ** 30)
            launches[k].append(ops.LAUNCHES - n0)
    nat.device_check()
    base = None
    for k in variants:
        ts = sorted(times[k])
        m = median(ts)
        base = m if base is None else base
        print(f"  {k:62s} median {m:8.1f} ms (min {ts[0]:.1f}, max {ts[-1]:.1f}, {len(ts)} steps, {100 * (m - base) / base:+.1f} %); "
              f"peak {median(peaks[k]):.2f} GiB; {median(launches[k])} launches", flush=True)


def bc_step(pol, opt, tr, batch, B):
    def step():
        opt.zero_grad()
        img, first, actions = batch
        tr.loss_and_grad(img, first, pol.initial_state(B), actions)
        opt.step()
    return step


def bc_2x():
    batch = frames(torch.Generator(device="cuda").manual_seed(0), 16)
    variants = {}
    for label, kw in (("all trainable", {}), ("CNN frozen (img_process.cnn.*)", dict(frozen=("net.img_process.cnn.",))),
                      ("below the transformer frozen (img_process.*)", dict(frozen=("net.img_process.",))),
                      ("heads only (pi_head.*)", dict(keep=("pi_head.",)))):
        pol, opt = policy(**kw)
        variants[f"2x BC B=16 T=128, {label}"] = bc_step(pol, opt, vpt_b200.BCTrainer(pol), batch, 16)
    timed(variants)


def big_2x():
    batch = frames(torch.Generator(device="cuda").manual_seed(1), 128)
    pol, opt = policy()
    pol_f, opt_f = policy(frozen=("net.img_process.cnn.",))
    timed({"2x BC B=128 T=128 one call, all trainable, recompute_frames=2048": bc_step(pol, opt, vpt_b200.BCTrainer(pol, recompute_frames=2048),
                                                                                         batch, 128),
           "2x BC B=128 T=128 one call, CNN frozen, no recompute": bc_step(pol_f, opt_f, vpt_b200.BCTrainer(pol_f), batch, 128)})


def rl_2x():
    g = torch.Generator(device="cuda").manual_seed(2)
    img, first, actions = frames(g, 16)
    old = -14.0 + 0.1 * torch.randn(16, T, device="cuda", generator=g)
    adv = torch.randn(16, T, device="cuda", generator=g)
    ret = 3.0 + torch.randn(16, T, device="cuda", generator=g)
    variants = {}
    for label, frozen in (("all trainable", ()), ("CNN frozen (img_process.cnn.*)", ("net.img_process.cnn.",))):
        pol, opt = policy(frozen=frozen, value_head=True)
        tr = vpt_b200.RLTrainer(pol)

        def step(pol=pol, opt=opt, tr=tr):
            opt.zero_grad()
            tr.loss_and_grad(img, first, pol.initial_state(16), actions, old, adv, ret, None, vf_coef=0.5, kl_coef=0.0)
            opt.step()
        variants[f"2x RL B=16 T=128, {label}"] = step
    timed(variants)


def main():
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    sections = dict(bc2x=bc_2x, big2x=big_2x, rl2x=rl_2x)
    for s in a.only.split(","):
        print(s, flush=True)
        sections[s]()
        gc.collect()  # (the step closures hold the section's policies)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
