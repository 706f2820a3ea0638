#!/usr/bin/env python
"""Truncated BPTT across calls (`set_autograd(True, state_grad=True)`) against the same window with the state detached between its chunks:
two chunks of B x 128 frames, the BC loss on both, ONE `loss.backward()` and `FlatAdamDP.step`, the two runs alternating in one process on
one GPU; then `vpt_attention_bwd_state` (state gradient in, memory gradient out) against `vpt_attention_bwd` at the same shape.

    python tools/bptt_bench.py [--width 2x] [--batch 8] [--steps 5] [--warmup 2]

Prints ms per step (CUDA events) and peak memory (`max_memory_allocated`, reset before each timed step) as medians over the steps, the
kernels' times, and the card's name and power limit read in the same run."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP

ap = argparse.ArgumentParser()
ap.add_argument("--width", default="2x")
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
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


def main():
    name, power = card()
    B = a.batch
    torch.manual_seed(0)
    kw = vpt_b200.policy_kwargs(a.width)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    chunks = []
    for _ in range(2):
        img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
        first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
        actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
                   "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
        chunks.append((img, first, actions))
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)
    state = {"bptt": pol.initial_state(B), "detached": pol.initial_state(B)}

    def step(kind):
        pol.set_autograd(True, state_grad=(kind == "bptt"))
        opt.zero_grad()
        st = [(m, (k.detach(), v.detach())) for m, (k, v) in state[kind]]  # truncation at the window start
        loss = 0.0
        for img, first, actions in chunks:
            (pd, _, _), st = pol({"img": img}, first, st)
            loss = loss - pol.logprob(actions, pd).mean()
            if kind == "detached":
                st = [(m, (k.detach(), v.detach())) for m, (k, v) in st]
        loss.backward()
        opt.step()
        state[kind] = st
        return loss

    for _ in range(a.warmup):
        for kind in ("bptt", "detached"):
            step(kind)
    torch.cuda.synchronize()
    nat.device_check()
    times = {"bptt": [], "detached": []}
    peak = {"bptt": [], "detached": []}
    for _ in range(a.steps):
        for kind in ("bptt", "detached"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = ev(), ev()
            e0.record()
            step(kind)
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1))
            peak[kind].append(torch.cuda.max_memory_allocated())
    nat.device_check()
    print(f"card: {name}, power limit {power}")
    for kind, label in (("bptt", "state attached (state_grad=True)"), ("detached", "state detached between the chunks")):
        ts = sorted(times[kind])
        print(f"{a.width} B={B} 2 x T={T}, BC loss on both, one backward + FlatAdamDP.step, {label:36s} median {median(ts):.1f} ms "
              f"(min {ts[0]:.1f}, max {ts[-1]:.1f}, {len(ts)} steps); peak {median(peak[kind]) / 2 ** 30:.2f} GiB")
    mb, md = median(times["bptt"]), median(times["detached"])
    print(f"BPTT overhead: {mb - md:+.1f} ms ({100 * (mb - md) / md:+.2f} %)")
    del state, opt
    kernel_bench(B, kw["attention_heads"], kw["attention_memory_size"] - T)


def kernel_bench(B, heads, maxlen, t=T, iters=50):
    """`attention_bwd` against `attention_bwd_state` with both state gradients given and the memory gradient written, CUDA events."""
    g = torch.Generator(device="cuda").manual_seed(1)
    h = heads * 128
    bf = lambda *s: torch.randn(*s, device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
    Q, Kf, Vf, dO = bf(B * t, h), bf(B, maxlen + t, h), bf(B, maxlen + t, h), bf(B * t, h)
    R = torch.randn(B * t, 10 * heads, device="cuda", generator=g)
    b_nd = torch.randn(10, maxlen, device="cuda", generator=g)
    first = torch.zeros(B, t, dtype=torch.uint8, device="cuda")
    smask = torch.ones(B, maxlen, dtype=torch.uint8, device="cuda")
    ds = (torch.randn(B, maxlen, h, device="cuda", generator=g), torch.randn(B, maxlen, h, device="cuda", generator=g))
    out = torch.zeros(B * t, (3 * h + 10 * heads + 7) // 8 * 8, dtype=torch.bfloat16, device="cuda")
    runs = {"attention_bwd": lambda: ops.attention_bwd(Q, Kf, Vf, R, b_nd, first, smask, dO, out, B, t, maxlen, heads),
            "attention_bwd_state": lambda: ops.attention_bwd_state(Q, Kf, Vf, R, b_nd, first, smask, dO, out, B, t, maxlen, heads, dstate=ds,
                                                                   want_dmem=True)}
    res = {}
    for _ in range(3):  # alternating rounds
        for n, fn in runs.items():
            for _ in range(5):
                fn()
            e0, e1 = ev(), ev()
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res.setdefault(n, []).append(e0.elapsed_time(e1) / iters)
    nat.device_check()
    for n, ts in res.items():
        print(f"{n:20s} B={B} t={t} maxlen={maxlen} heads={heads}: median {median(ts) * 1e3:.1f} us per call (3 rounds of {iters}, "
              f"buffers allocated inside the call included)")


if __name__ == "__main__":
    main()
