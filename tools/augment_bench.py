#!/usr/bin/env python
"""Training-time augmentation (`augment_frames`, `vpt_augment_frames`): kernel time against its HBM bound, and the 2x BC step with and
without it.

    python tools/augment_bench.py [--frames 2048] [--reps 50] [--steps 5] [--warmup 2]

    kernel  device time (CUDA events over `--reps` launches, median of five windows) of `augment_frames` for `--frames` frames at
            128 x 128 with every step active (rotate, scale, shear, translate, brightness, contrast, saturation, hue), with uint8 and
            with fp32 output, against the HBM bound of reading the frames once and writing the output once (3.35 TB/s, the H100 SXM data
            sheet's HBM3 bandwidth); the same with identity colour factors (warp only: no contrast pass, no hue)
    bc2x    2x BC at B = 16, T = 128 (BCTrainer + FlatAdamDP.step): un-augmented frames against augment_frames(img, augment_params(B))
            with per-sequence draws, uint8 output; medians of alternating steps, each step drawing new parameters

The card's name and power limit are read in the same run."""
import argparse
import os
import subprocess
import sys

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import _native as nat
from video_pre_training_b200.parallel import FlatAdamDP

ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=2048)
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--only", default="kernel,bc2x")
a = ap.parse_args()
HBM = 3.35e12
JITTER = dict(rotate=10.0, scale=(0.9, 1.1), shear=5.0, translate=8.0, brightness=(0.8, 1.2), contrast=(0.8, 1.2), saturation=(0.8, 1.2),
              hue=0.05)
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


def kernel():
    from video_pre_training_b200 import ops
    from video_pre_training_b200.agent import augment_rows

    F_ = a.frames
    g = torch.Generator().manual_seed(0)
    img = torch.randint(0, 256, (F_, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    full = vpt_b200.augment_params(F_, generator=g, **JITTER)
    warp = full.clone()
    warp[:, 5:9] = torch.tensor([1.0, 1.0, 1.0, 0.0])
    for label, p in (("all steps", full), ("warp only", warp)):
        rows = torch.from_numpy(augment_rows(p, img.shape)).cuda()
        for dt in (torch.uint8, torch.float32):
            out = torch.empty(img.shape, dtype=dt, device="cuda")
            for _ in range(3):
                ops.augment(img, rows, out)
            torch.cuda.synchronize()
            nat.device_check()
            windows = []
            for _ in range(5):
                e0, e1 = ev(), ev()
                e0.record()
                for _ in range(a.reps):
                    ops.augment(img, rows, out)
                e1.record()
                torch.cuda.synchronize()
                windows.append(e0.elapsed_time(e1) * 1e3 / a.reps)
            us = median(windows)
            nbytes = img.numel() * (1 + out.element_size())
            bound = nbytes / HBM * 1e6
            print(f"  augment_frames {F_} x 128x128, {label:9s}, {str(dt).replace('torch.', ''):7s} out: median {us:7.1f} us "
                  f"(windows {min(windows):.1f}-{max(windows):.1f}); HBM bound {bound:.1f} us ({nbytes / 1e6:.0f} MB) -> {bound / us:.2f} of it",
                  flush=True)


def bc2x():
    B, T = 16, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
               "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)
    tr = vpt_b200.BCTrainer(pol)
    pg = torch.Generator().manual_seed(1)

    def step(augment):
        opt.zero_grad()
        x = vpt_b200.augment_frames(img, vpt_b200.augment_params(B, generator=pg, **JITTER)) if augment else img
        tr.loss_and_grad(x, first, pol.initial_state(B), actions)
        opt.step()

    variants = {"2x BC B=16 T=128, no augmentation": lambda: step(False), "2x BC B=16 T=128, augment_frames per sequence": lambda: step(True)}
    for _ in range(a.warmup):
        for fn in variants.values():
            fn()
    torch.cuda.synchronize()
    nat.device_check()
    times = {k: [] for k in variants}
    for _ in range(a.steps):
        for k, fn in variants.items():
            torch.cuda.synchronize()
            e0, e1 = ev(), ev()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    nat.device_check()
    base = None
    for k, ts in times.items():
        m = median(ts)
        base = m if base is None else base
        print(f"  {k:50s} median {m:8.1f} ms (min {min(ts):.1f}, max {max(ts):.1f}, {len(ts)} steps, {100 * (m - base) / base:+.1f} %)", flush=True)


if __name__ == "__main__":
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    only = a.only.split(",")
    if "kernel" in only:
        kernel()
    if "bc2x" in only:
        bc2x()
