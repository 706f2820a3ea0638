#!/usr/bin/env python
"""Entropy and KL on the action heads (csrc/head_dist.cuh, `pi_head.entropy` / `pi_head.kl_divergence`) and the RL entropy bonus, on one
GPU.  Prints the card's name and power limit from the same run, then

  - each head distribution kernel's device time (CUDA events around a CUDA graph of many calls, so no host enqueue time) at the 2x
    RL / BC call shape, N = 2048 rows of each agent head (121 and 8641 columns) and of both, against the HBM bound computed from the
    shapes at the H100 SXM data-sheet 3.35 TB/s;
  - the 2x RL step at B = 16, T = 128 (RLTrainer.loss_and_grad + FlatAdamDP.step), ent_coef 0 against 0.01, alternating, medians;
  - the 2x `loss.backward()` BC step with an entropy bonus, B = 16, T = 128: `pi_head.entropy(pd)` against the torch-op formula
    -(exp(lp) * lp).sum(-1), alternating, medians and peak memory.

    python tools/head_dist_bench.py [--steps 5] [--warmup 2] [--reps 50]"""
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth
HEADS = (121, 8641)

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=16)
ap.add_argument("--T", type=int, default=128)
ap.add_argument("--steps", type=int, default=5, help="timed steps per variant (alternating)")
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--reps", type=int, default=50, help="launches per kernel timing")
a = ap.parse_args()
B, T = a.B, a.T
N = B * T


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def ev():
    return torch.cuda.Event(enable_timing=True)


def kernel_time(fn):
    """us per call of `fn` from a CUDA graph of `reps` calls: device time only, without the wrappers' host-side enqueue."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(a.reps):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = ev(), ev()
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    del graph
    return e0.elapsed_time(e1) / a.reps * 1e3


def kernels():
    """Per kernel and head: device time against the bytes it must move (each operand read once, each result written once)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    lp = {n: torch.log_softmax(3 * torch.randn(N, n, device="cuda", generator=g), -1) for n in HEADS}
    lq = {n: torch.log_softmax(3 * torch.randn(N, n, device="cuda", generator=g), -1) for n in HEADS}
    up = torch.randn(N, device="cuda", generator=g)
    # name -> (call on head n, full-width fp32 arrays read + written)
    rows = {"entropy forward": (lambda n: ops.head_entropy(lp[n]), 1),
            "KL forward": (lambda n: ops.head_kl(lq[n], lp[n]), 2),
            "entropy backward": (lambda n: ops.head_entropy_bwd(lp[n], up), 2),
            "KL backward, d logp only": (lambda n: ops.head_kl_bwd(lq[n], lp[n], up, want_q=False), 3),
            "KL backward, both sides": (lambda n: ops.head_kl_bwd(lq[n], lp[n], up), 4)}
    print(f"head distribution kernels at N = {N} rows, per head and for both ({' + '.join(map(str, HEADS))} columns); device time per call "
          f"from a CUDA graph of {a.reps} calls:")
    for name, (fn, arrays) in rows.items():
        parts = []
        for n in HEADS + (None,):
            if n is None:
                us, nbytes, label = sum(p[1] for p in parts), sum(p[2] for p in parts), "both"
            else:
                us, nbytes, label = kernel_time(lambda n=n: fn(n)), N * n * 4 * arrays + N * 4, f"n={n}"
                parts.append((n, us, nbytes))
            bound = nbytes / HBM_BYTES_PER_S * 1e6
            print(f"  {name:26s} {label:7s} {us:7.1f} us  {nbytes / 1e6:6.1f} MB  {nbytes / (us * 1e-6) / 1e12:5.2f} TB/s  "
                  f"(HBM bound {bound:.1f} us at 3.35 TB/s: {bound / us * 100:.0f} % of it)")
        torch.cuda.empty_cache()
    nat.device_check()


def setup():
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
               "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
    return pol, g, img, first, actions


def alternate(step, variants, after=None):
    """Warm-up, then `a.steps` rounds of one step per variant; `after(v)` runs outside the timed window after each step."""
    for _ in range(a.warmup):
        for v in variants:
            step(v)
    torch.cuda.synchronize()
    nat.device_check()
    times, peak = {v: [] for v in variants}, {v: 0 for v in variants}
    for _ in range(a.steps):
        for v in variants:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = ev(), ev()
            e0.record()
            step(v)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1))
            peak[v] = max(peak[v], torch.cuda.max_memory_allocated())
            if after is not None:
                after(v)
    return {v: sorted(ts) for v, ts in times.items()}, peak


def report(label, ts, peak):
    print(f"  {label:44s} median {ts[len(ts) // 2]:7.1f} ms (min {ts[0]:.1f}, max {ts[-1]:.1f}, {len(ts)} steps); peak {peak / 2 ** 30:.2f} GiB")


def rl_steps():
    pol, g, img, first, actions = setup()
    with torch.no_grad():
        (pd_ref, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
    old = pol.logprob(actions, pd_ref).reshape(B, T).float() + 0.1 * torch.randn(B, T, device="cuda", generator=g)
    adv = torch.randn(B, T, device="cuda", generator=g)
    returns = 3.0 + torch.randn(B, T, device="cuda", generator=g)
    tr = vpt_b200.RLTrainer(pol)
    opt = FlatAdamDP([p for p in pol.parameters() if p.requires_grad], lr=1e-5)
    stats = {}

    def step(ent_coef):
        opt.zero_grad()
        tr.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, vf_coef=0.5, kl_coef=0.1, ent_coef=ent_coef)
        opt.step()

    def read_entropy(ent_coef):  # (outside the timing: with ent_coef 0 the entropy is computed when first read)
        stats[ent_coef] = tr.stats["entropy"].item()

    times, peak = alternate(step, (0.0, 0.01), read_entropy)
    print(f"2x RL step, B={B} T={T}: RLTrainer.loss_and_grad + FlatAdamDP.step (pd_ref precomputed)")
    for v in (0.0, 0.01):
        report(f"ent_coef {v} (entropy {stats[v]:.4f})", times[v], peak[v])
    m0, m1 = times[0.0][len(times[0.0]) // 2], times[0.01][len(times[0.01]) // 2]
    print(f"  entropy bonus: {m1 - m0:+.2f} ms ({100 * (m1 - m0) / m0:+.2f} %)")


def bc_steps():
    pol, _, img, first, actions = setup()
    pol.set_autograd(True)
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=1e-5)

    def step(kind):
        opt.zero_grad()
        (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
        if kind == "kernels":
            ent = pol.pi_head.entropy(pd)
        else:  # the torch-op formula
            ent = sum(-(torch.exp(v) * v).sum(-1).sum(-1) for v in pd.values())
        (-pol.logprob(actions, pd).mean() - 0.01 * ent.mean()).backward()
        opt.step()

    times, peak = alternate(step, ("kernels", "torch ops"))
    print(f"2x loss.backward() BC step with an entropy bonus, B={B} T={T}: (nll - 0.01 * mean H).backward() + FlatAdamDP.step")
    report("pi_head.entropy(pd)", times["kernels"], peak["kernels"])
    report("-(exp(lp) * lp).sum(-1) in torch ops", times["torch ops"], peak["torch ops"])
    mk, mt = times["kernels"][len(times["kernels"]) // 2], times["torch ops"][len(times["torch ops"]) // 2]
    print(f"  kernels against torch ops: {mk - mt:+.2f} ms, peak {(peak['kernels'] - peak['torch ops']) / 2 ** 20:+.0f} MiB")


def main():
    name, power = card()
    print(f"card: {name}, power limit {power}")
    kernels()
    rl_steps()
    torch.cuda.empty_cache()
    bc_steps()


if __name__ == "__main__":
    main()
