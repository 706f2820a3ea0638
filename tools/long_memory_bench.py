#!/usr/bin/env python
"""The cost of a longer KV memory at 2x width: attention_memory_size 256 (maxlen 128, the released models) against 2048 (maxlen 1920, the
reference's default), the two alternating in one process on one GPU.

    python tools/long_memory_bench.py [--steps 5] [--warmup 2]

  forward   B x T = 128 x 128 inference chunks with the state carried from chunks that filled the memory: frames/s, and the attention
            kernels' time (torch.profiler) with their achieved TFLOP/s over the band's FLOPs (4 h maxlen + 2 * 10 heads maxlen per frame and
            layer, counted here)
  bc        BCTrainer.loss_and_grad + FlatAdamDP.step at B = 16, T = 128: ms and peak memory
  bptt      (maxlen 1920) a window of two B = 8, T = 128 chunks, `loss.backward()` with the state attached + FlatAdamDP.step
  rollout   GraphedAct at B = 1 and B = 64: ms per step, and the bytes a step must move (bf16 weights + the KV state read and written)
            against the HBM bound (3.35 TB/s)

Medians over the timed steps (CUDA events); the card's name and power limit are read in the same run."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200.parallel import FlatAdamDP
from video_pre_training_b200.policy import GraphedAct
from video_pre_training_b200.training import BCTrainer

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
a = ap.parse_args()
T = 128
SIZES = (256, 2048)
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


def policy(ams):
    torch.manual_seed(0)
    kw = vpt_b200.policy_kwargs("2x", attention_memory_size=ams)
    return vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS).cuda()


def timed(fn):
    e0, e1 = ev(), ev()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def frames(g, B, t):
    return (torch.randint(0, 256, (B, t, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g),
            torch.zeros(B, t, dtype=torch.bool, device="cuda"))


def bench_forward(pols):
    B = 128
    g = torch.Generator(device="cuda").manual_seed(0)
    img, first = frames(g, B, T)
    states = {}
    with torch.no_grad():
        for ams, pol in pols.items():
            st = pol.initial_state(B)
            for _ in range((pol.net.cfg.maxlen + T - 1) // T):  # fill the memory
                _, st = pol({"img": img}, first, st)
            states[ams] = st
        ms = {ams: [] for ams in pols}
        for it in range(a.warmup + a.steps):
            for ams, pol in pols.items():
                t = timed(lambda: pol({"img": img}, first, states[ams]))
                if it >= a.warmup:
                    ms[ams].append(t)
        out = {}
        for ams, pol in pols.items():
            cfg = pol.net.cfg
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                pol({"img": img}, first, states[ams])
                torch.cuda.synchronize()
            att = sum(e.device_time_total for e in prof.key_averages() if "attention" in e.key) / 1e3  # ms
            copies = sum(e.device_time_total for e in prof.key_averages() if "copy_rows" in e.key) / 1e3
            flops = cfg.n_layers * B * T * (4 * cfg.hidsize * cfg.maxlen + 2 * 10 * cfg.heads * cfg.maxlen)
            m = median(ms[ams])
            out[ams] = dict(maxlen=cfg.maxlen, ms=round(m, 2), frames_per_s=round(B * T / m * 1e3), attention_ms=round(att, 3),
                            attention_tflops=round(flops / (att * 1e-3) / 1e12, 1), kv_copy_ms=round(copies, 3))
        del states
    return out


def bench_bc(pols):
    B = 16
    g = torch.Generator(device="cuda").manual_seed(1)
    img, first = frames(g, B, T)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
               "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
    runs = {ams: (BCTrainer(pol), FlatAdamDP([p for p in pol.parameters() if p.requires_grad], lr=1e-6)) for ams, pol in pols.items()}
    ms, peak = {ams: [] for ams in pols}, {ams: [] for ams in pols}
    for it in range(a.warmup + a.steps):
        for ams, pol in pols.items():
            tr, opt = runs[ams]
            torch.cuda.reset_peak_memory_stats()

            def step():
                opt.zero_grad()
                tr.loss_and_grad(img, first, pol.initial_state(B), actions)
                opt.step()
            t = timed(step)
            if it >= a.warmup:
                ms[ams].append(t)
                peak[ams].append(torch.cuda.max_memory_allocated() / 2**30)
    for ams, pol in pols.items():
        pol.zero_grad(set_to_none=True)
    out = {ams: dict(ms=round(median(ms[ams]), 1), peak_gib=round(median(peak[ams]), 2)) for ams in pols}
    del runs
    return out


def bench_bptt(pol):
    B = 8
    g = torch.Generator(device="cuda").manual_seed(2)
    chunks = []
    for _ in range(2):
        img, first = frames(g, B, T)
        chunks.append((img, first, {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
                                    "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}))
    pol.set_autograd(True, state_grad=True)
    opt = FlatAdamDP([p for p in pol.parameters() if p.requires_grad], lr=1e-6)
    ms, peak = [], []
    for it in range(a.warmup + a.steps):
        torch.cuda.reset_peak_memory_stats()

        def step():
            opt.zero_grad()
            st, loss = pol.initial_state(B), 0.0
            for img, first, actions in chunks:
                (pd, _, _), st = pol({"img": img}, first, st)
                loss = loss - pol.logprob(actions, pd).mean()
            loss.backward()
            opt.step()
        t = timed(step)
        if it >= a.warmup:
            ms.append(t)
            peak.append(torch.cuda.max_memory_allocated() / 2**30)
    pol.set_autograd(False)
    pol.zero_grad(set_to_none=True)
    del opt
    return dict(maxlen=pol.net.cfg.maxlen, ms=round(median(ms), 1), peak_gib=round(median(peak), 2))


def bench_rollout(pols, B):
    g = torch.Generator(device="cuda").manual_seed(3)
    obs = {"img": torch.randint(0, 256, (B, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)}
    first = torch.zeros(B, dtype=torch.bool, device="cuda")
    acts = {ams: GraphedAct(pol, B) for ams, pol in pols.items()}
    states = {ams: pol.initial_state(B) for ams, pol in pols.items()}
    n = 20
    ms = {ams: [] for ams in pols}
    for it in range(a.warmup + a.steps):
        for ams in pols:
            def run():
                st = states[ams]
                for _ in range(n):
                    _, st, _ = acts[ams](obs, first, st)
                states[ams] = st
            t = timed(run) / n
            if it >= a.warmup:
                ms[ams].append(t)
    out = {}
    for ams, pol in pols.items():
        cfg = pol.net.cfg
        wbytes = 2 * sum(p.numel() for p in pol.parameters())
        h, L = cfg.hidsize, cfg.n_layers
        kv = L * B * h * (2 * cfg.maxlen * 4 * 2 + 2 * (cfg.maxlen + 1) * 2 * 2)  # fp32 state in + out, bf16 [memory|chunk] written + read
        m = median(ms[ams])
        out[ams] = dict(ms=round(m, 3), weight_mb=round(wbytes / 1e6, 1), kv_mb=round(kv / 1e6, 1),
                        hbm_bound_ms=round((wbytes + kv) / HBM * 1e3, 3))
    del acts, states
    return out


def main():
    name, power = card()
    pols = {ams: policy(ams) for ams in SIZES}
    res = dict(card=name, power_limit=power, forward_B128=bench_forward(pols))
    torch.cuda.empty_cache()
    res["bc_B16"] = bench_bc(pols)
    torch.cuda.empty_cache()
    res["bptt_2x_B8"] = bench_bptt(pols[2048])
    torch.cuda.empty_cache()
    res["rollout_B1"] = bench_rollout(pols, 1)
    res["rollout_B64"] = bench_rollout(pols, 64)
    import json

    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
