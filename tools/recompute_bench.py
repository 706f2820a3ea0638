#!/usr/bin/env python
"""`recompute_frames` (the backward re-runs the ImpalaCNN chunk by chunk) against the stored CNN tape: ms per training step and peak memory.

    python tools/recompute_bench.py [--steps 3] [--warmup 1] [--only bc2x,big2x,bc3x,bptt3x,idm4x]

    bc2x    2x BC at B = 16, T = 128 (BCTrainer + FlatAdamDP.step): stored tape against recompute_frames = 2048 and 512, alternating rounds
    big2x   2x BC at B = 128, T = 128 in ONE call with recompute_frames = 2048, against eight accumulated stored-tape B = 16 calls
    bc3x    3x BC at B = 16, T = 128: stored tape against recompute_frames = 512
    bptt3x  3x truncated-BPTT window (`loss.backward()`, state_grad) of k = 2 and 4 calls of B = 16, T = 128, recompute_frames = 512
    idm4x   the 4x IDM at B = 16, T = 128 in one call with recompute_frames = 512, against four accumulated stored-tape B = 4 calls

Times are CUDA events around the whole step (medians over the timed steps, the variants alternating), peak memory is
`max_memory_allocated` reset before each timed step.  The card's name and power limit are read in the same run.  The 3x stored tape at
B = 16 needs nearly all of an 80 GB card: run bc3x in a process of its own (--only bc3x); the allocator's expandable segments keep
fragmentation from costing it the last few GiB."""
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
from video_pre_training_b200.parallel import FlatAdamDP

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--only", default="bc2x,big2x,bc3x,bptt3x,idm4x")
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


def policy(width):
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS).cuda()
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)
    return pol, opt


def timed(variants):
    """variants: {label: step function}; warm-up, then alternating timed rounds -> {label: (median ms, min, max, median peak GiB)}."""
    for _ in range(a.warmup):
        for fn in variants.values():
            fn()
    torch.cuda.synchronize()
    nat.device_check()
    times, peaks = {k: [] for k in variants}, {k: [] for k in variants}
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
    out = {}
    for k in variants:
        ts = sorted(times[k])
        out[k] = (median(ts), ts[0], ts[-1], median(peaks[k]))
        print(f"  {k:60s} median {out[k][0]:8.1f} ms (min {ts[0]:.1f}, max {ts[-1]:.1f}, {len(ts)} steps); peak {out[k][3]:.2f} GiB", flush=True)
    return out


def bc_step(pol, opt, trainers, batches, B):
    def step():
        opt.zero_grad()
        for tr, (img, first, actions) in zip(trainers, batches):
            tr.loss_and_grad(img, first, pol.initial_state(B), actions)
        opt.step()
    return step


def bc_stored_vs_recompute(width, rfs):
    pol, opt = policy(width)
    batch = [frames(torch.Generator(device="cuda").manual_seed(0), 16)]
    tr = vpt_b200.BCTrainer(pol)

    def with_recompute(rf):
        step = bc_step(pol, opt, [tr], batch, 16)

        def run():
            tr.recompute_frames = rf
            step()
        return run
    variants = {f"{width} BC B=16 T=128, stored CNN tape": with_recompute(None)}
    for rf in rfs:
        variants[f"{width} BC B=16 T=128, recompute_frames={rf}"] = with_recompute(rf)
    res = list(timed(variants).items())
    s = res[0][1][0]
    for k, v in res[1:]:
        print(f"  {k}: recompute overhead {v[0] - s:+.1f} ms ({100 * (v[0] - s) / s:+.1f} %)", flush=True)


def big_2x():
    pol, opt = policy("2x")
    g = torch.Generator(device="cuda").manual_seed(1)
    parts = [frames(g, 16) for _ in range(8)]
    big = (torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]), {k: torch.cat([p[2][k] for p in parts]) for k in parts[0][2]})
    stored = vpt_b200.BCTrainer(pol)
    timed({"2x BC 8 x (B=16, T=128) stored-tape calls accumulated, one step": bc_step(pol, opt, [stored] * 8, parts, 16),
           "2x BC B=128 T=128 one call, recompute_frames=2048, one step": bc_step(pol, opt, [vpt_b200.BCTrainer(pol, recompute_frames=2048)],
                                                                                   [big], 128)})


def bptt_3x():
    pol, opt = policy("3x")
    pol.set_autograd(True, state_grad=True, recompute_frames=512)
    g = torch.Generator(device="cuda").manual_seed(2)
    chunks = [frames(g, 16) for _ in range(4)]

    def window(k):
        def step():
            opt.zero_grad()
            st, loss = pol.initial_state(16), 0.0
            for img, first, actions in chunks[:k]:
                (pd, _, _), st = pol({"img": img}, first, st)
                loss = loss - pol.logprob(actions, pd).mean()
            loss.backward()
            opt.step()
        return step
    timed({f"3x BPTT window of {k} x (B=16, T=128), recompute_frames=512, one backward + step": window(k) for k in (2, 4)})


def idm_4x():
    torch.manual_seed(0)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()
    opt = FlatAdamDP(vpt_b200.IDMTrainer.optimizer_params(pol), lr=1e-5)
    g = torch.Generator(device="cuda").manual_seed(3)
    img = torch.randint(0, 256, (16, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    first = torch.zeros(16, T, dtype=torch.bool, device="cuda")
    actions = {"buttons": torch.randint(0, 2, (16, T, 20), device="cuda", generator=g),
               "camera": torch.randint(0, 11, (16, T, 2), device="cuda", generator=g)}
    parts = [(img[b:b + 4], first[b:b + 4], {k: v[b:b + 4] for k, v in actions.items()}) for b in range(0, 16, 4)]
    stored = vpt_b200.IDMTrainer(pol)
    timed({"4x IDM 4 x (B=4, T=128) stored-tape calls accumulated, one step": bc_step(pol, opt, [stored] * 4, parts, 4),
           "4x IDM B=16 T=128 one call, recompute_frames=512, one step": bc_step(pol, opt, [vpt_b200.IDMTrainer(pol, recompute_frames=512)],
                                                                                  [(img, first, actions)], 16)})


def main():
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    sections = dict(bc2x=lambda: bc_stored_vs_recompute("2x", (2048, 512)), big2x=big_2x, bc3x=lambda: bc_stored_vs_recompute("3x", (512,)),
                    bptt3x=bptt_3x, idm4x=idm_4x)
    for s in a.only.split(","):
        print(s, flush=True)
        sections[s]()
        gc.collect()  # (the step closures and the trainers hold the section's policy in reference cycles)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
