#!/usr/bin/env python
"""Training from cached CNN latents (`encode`, then `loss_and_grad(latents, ...)`) against training from frames: ms per step, peak memory.

    python tools/latent_bench.py [--steps 5] [--warmup 1] [--only bc2x,big2x,rl2x,idm4x]

    bc2x    2x BC at B = 16, T = 128 (BCTrainer + FlatAdamDP.step): all trainable from frames, the CNN (`img_process.cnn.*`) frozen from
            frames, and from latents; and `encode` of those 2048 frames
    big2x   2x BC at B = 128, T = 128 in one call from latents (no recompute_frames)
    rl2x    the 2x RL step at B = 16, T = 128 (RLTrainer with kl_coef = 0.1 + FlatAdamDP.step), the CNN frozen, from frames against from
            latents; both count the frozen reference policy's forward for pd_ref on the same input (frames / latents)
    idm4x   the 4x IDM at B = 4, T = 128 (IDMTrainer + FlatAdamDP.step), the CNN and conv3d pre-stage frozen, from frames against from latents

Times are CUDA events around the whole step (medians over the timed steps, the variants alternating), peak memory is
`max_memory_allocated` reset before each timed step.  Every training variant has its own policy (the same seed) and its own FlatAdamDP
over its trainable parameters.  The latents are encoded once, outside the timed steps (as a multi-epoch run would), with the weights the
step starts from: the frozen CNN does not change.  The card's name, power limit and SM clocks are read in the same run."""
import argparse
import copy
import gc
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
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--only", default="bc2x,big2x,rl2x,idm4x")
a = ap.parse_args()
T = 128
CNN = ("net.img_process.cnn.", "net.conv3d_layer.")
ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        info = "unknown"
    return name, info


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def frames(g, B):
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
               "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
    return img, torch.zeros(B, T, dtype=torch.bool, device="cuda"), actions


def policy(frozen=(), value_head=False):
    """The 2x policy with the parameters under `frozen` frozen, and its optimizer over the trainable ones."""
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
    for n, p in pol.named_parameters():
        if n.startswith(tuple(frozen)):
            p.requires_grad_(False)
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if value_head or not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)
    return pol, opt


def timed(variants):
    """variants: {label: step function}; warm-up, then alternating timed rounds; prints median ms and peak GiB per step."""
    for _ in range(a.warmup):
        for fn in variants.values():
            fn()
    torch.cuda.synchronize()
    nat.device_check()
    times, peaks = ({k: [] for k in variants} for _ in range(2))
    for _ in range(a.steps):
        for k, fn in variants.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = ev(), ev()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            peaks[k].append(torch.cuda.max_memory_allocated() / 2 ** 30)
    nat.device_check()
    base = None
    for k in variants:
        ts = sorted(times[k])
        m = median(ts)
        base = m if base is None else base
        print(f"  {k:66s} median {m:8.1f} ms (min {ts[0]:.1f}, max {ts[-1]:.1f}, {len(ts)} steps, {100 * (m - base) / base:+.1f} %); "
              f"peak {median(peaks[k]):.2f} GiB", flush=True)


def bc_step(pol, opt, tr, x, first, actions):
    B = first.shape[0]

    def step():
        opt.zero_grad()
        tr.loss_and_grad(x, first, pol.initial_state(B), actions)
        opt.step()
    return step


def bc_2x():
    img, first, actions = frames(torch.Generator(device="cuda").manual_seed(0), 16)
    pol_a, opt_a = policy()
    pol_f, opt_f = policy(frozen=CNN)
    pol_l, opt_l = policy(frozen=CNN)
    lat = pol_l.encode(img)
    timed({"2x BC B=16 T=128, all trainable, from frames": bc_step(pol_a, opt_a, vpt_b200.BCTrainer(pol_a), img, first, actions),
           "2x BC B=16 T=128, CNN frozen, from frames": bc_step(pol_f, opt_f, vpt_b200.BCTrainer(pol_f), img, first, actions),
           "2x BC B=16 T=128, from latents": bc_step(pol_l, opt_l, vpt_b200.BCTrainer(pol_l), lat, first, actions),
           "encode 16 x 128 frames (2x)": lambda: pol_l.encode(img)})


def big_2x():
    img, first, actions = frames(torch.Generator(device="cuda").manual_seed(1), 128)
    pol, opt = policy(frozen=CNN)
    lat = pol.encode(img)
    del img
    torch.cuda.empty_cache()
    timed({"2x BC B=128 T=128 one call, from latents": bc_step(pol, opt, vpt_b200.BCTrainer(pol), lat, first, actions)})


def rl_2x():
    g = torch.Generator(device="cuda").manual_seed(2)
    img, first, actions = frames(g, 16)
    old = -14.0 + 0.1 * torch.randn(16, T, device="cuda", generator=g)
    adv = torch.randn(16, T, device="cuda", generator=g)
    ret = 3.0 + torch.randn(16, T, device="cuda", generator=g)
    variants = {}
    for label in ("frames", "latents"):
        pol, opt = policy(frozen=CNN, value_head=True)
        ref = copy.deepcopy(pol).requires_grad_(False)  # the frozen reference policy: the same pretrained CNN
        tr = vpt_b200.RLTrainer(pol)
        x, key = (img, "img") if label == "frames" else (pol.encode(img), "img_latent")

        def step(pol=pol, opt=opt, tr=tr, ref=ref, x=x, key=key):
            opt.zero_grad()
            with torch.no_grad():
                (pd_ref, _, _), _ = ref({key: x}, first, ref.initial_state(16))
            tr.loss_and_grad(x, first, pol.initial_state(16), actions, old, adv, ret, pd_ref, vf_coef=0.5, kl_coef=0.1)
            opt.step()
        variants[f"2x RL B=16 T=128 + reference forward, CNN frozen, from {label}"] = step
    timed(variants)


def idm_4x():
    g = torch.Generator(device="cuda").manual_seed(3)
    img = torch.randint(0, 256, (4, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    first = torch.zeros(4, T, dtype=torch.bool, device="cuda")
    actions = {"buttons": torch.randint(0, 2, (4, T, 20), device="cuda", generator=g),
               "camera": torch.randint(0, 11, (4, T, 2), device="cuda", generator=g)}
    variants = {}
    for label in ("frames", "latents"):
        torch.manual_seed(0)
        idm = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()
        for n, p in idm.named_parameters():
            if n.startswith(CNN):
                p.requires_grad_(False)
        opt = FlatAdamDP(vpt_b200.IDMTrainer.optimizer_params(idm), lr=0.000181, weight_decay=0.039428)
        x = img if label == "frames" else idm.encode(img)
        variants[f"4x IDM B=4 T=128, CNN + conv3d frozen, from {label}"] = bc_step(idm, opt, vpt_b200.IDMTrainer(idm), x, first, actions)
    timed(variants)


def main():
    name, info = card()
    print(f"card: {name}, power limit / max SM clock / SM clock: {info}", flush=True)
    sections = dict(bc2x=bc_2x, big2x=big_2x, rl2x=rl_2x, idm4x=idm_4x)
    for s in a.only.split(","):
        print(s, flush=True)
        sections[s]()
        gc.collect()  # (the step closures hold the section's policies)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
