#!/usr/bin/env python
"""The BC step through `BCTrainer.loss_and_grad` against the same loss through the differentiable forward (`set_autograd` +
`loss.backward()`), both finished by `FlatAdamDP.step`, alternating in one run on one GPU; then `log_softmax_bwd` against its HBM bound,
and one autograd step at a second width to show it fits.

    python tools/autograd_bench.py [--width 2x] [--batch 16] [--steps 5] [--warmup 3] [--fit-width 3x] [--ops]

Prints ms per step (CUDA events) and peak memory (`max_memory_allocated`, reset before each path's timed steps) for both paths, the
kernel's time and bandwidth, and the card's name and power limit read in the same run."""
import argparse
import gc
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.parallel import FlatAdamDP
from video_pre_training_b200.training import BCTrainer

ap = argparse.ArgumentParser()
ap.add_argument("--width", default="2x")
ap.add_argument("--fit-width", default="3x", help="width run once through the autograd path to report its peak memory ('' to skip)")
ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--ops", action="store_true", help="per-op CUDA-event breakdown of one step of each path")
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


def setup(width, B):
    torch.manual_seed(0)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
    first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
               "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
    opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)
    return pol, img, first, actions, opt


def autograd_loss(pol, img, first, state, actions):
    """behavioural_cloning.py:101-123's loss for a whole batch: -mean log p(action) over the B*T frames."""
    (pd, _, _), state = pol({"img": img}, first, state)
    return -pol.logprob(actions, pd).mean(), state


def main():
    name, power = card()
    B = a.batch
    pol, img, first, actions, opt = setup(a.width, B)
    tr = BCTrainer(pol)
    pol.set_autograd(True)
    st = {"bc": pol.initial_state(B), "ag": pol.initial_state(B)}

    def step(kind):
        opt.zero_grad()
        if kind == "bc":
            loss, st[kind] = tr.loss_and_grad(img, first, st[kind], actions)
        else:
            loss, st[kind] = autograd_loss(pol, img, first, st[kind], actions)
            loss.backward()
        opt.step()
        return loss

    for _ in range(a.warmup):
        for kind in ("bc", "ag"):
            step(kind)
    torch.cuda.synchronize()
    nat.device_check()
    times = {"bc": [], "ag": []}
    peak = {"bc": 0, "ag": 0}
    for _ in range(a.steps):
        for kind in ("bc", "ag"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = ev(), ev()
            e0.record()
            step(kind)
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1))
            peak[kind] = max(peak[kind], torch.cuda.max_memory_allocated())
    print(f"card: {name}, power limit {power}")
    for kind, label in (("bc", "BCTrainer.loss_and_grad + FlatAdamDP.step"), ("ag", "set_autograd + loss.backward() + FlatAdamDP.step")):
        ts = sorted(times[kind])
        print(f"{a.width} B={B} T={T}  {label:50s} median {ts[len(ts) // 2]:.1f} ms (min {ts[0]:.1f}, max {ts[-1]:.1f}, {len(ts)} steps); "
              f"peak {peak[kind] / 2 ** 30:.2f} GiB")
    mb, ma = sorted(times["bc"])[len(times["bc"]) // 2], sorted(times["ag"])[len(times["ag"]) // 2]
    print(f"autograd overhead: {ma - mb:+.1f} ms ({100 * (ma - mb) / mb:+.2f} %)")
    if a.ops:
        breakdown(pol, tr, img, first, actions, opt, st)
    del tr, opt, st
    kernel_bench()
    if a.fit_width:
        del pol, step
        gc.collect()  # (a policy and its differentiable-forward runner reference each other)
        torch.cuda.empty_cache()
        fit(a.fit_width, B)


def breakdown(pol, tr, img, first, actions, opt, st):
    """CUDA-event time per op of one step of each path (outer ops include those they call), and the time outside them."""
    import collections

    names = [n for n in ("gemm", "conv3x3_zp", "wgrad", "firstconv_pool", "maxpool3s2", "affine_norm", "affine_norm_zp", "add_zp", "attention",
                         "relu_mask", "group_sums", "col_sums", "norm_sums", "norm_bwd_apply", "maxpool3s2_bwd", "firstconv_bwd", "attention_bwd",
                         "softmax_bwd", "log_softmax_bwd", "copy_rows", "copy_rows2", "log_softmax", "gather_logprob", "stats_finalize")
             if hasattr(ops, n)]
    saved = {n: getattr(ops, n) for n in names}
    for kind in ("bc", "ag"):
        rec = []

        def wrap(n, f):
            def gfn(*args, **kw):
                e0, e1 = ev(), ev()
                e0.record()
                r = f(*args, **kw)
                e1.record()
                rec.append((n, e0, e1))
                return r
            return gfn

        for n in names:
            setattr(ops, n, wrap(n, saved[n]))
        try:
            opt.zero_grad()
            s0, s1 = ev(), ev()
            s0.record()
            if kind == "bc":
                tr.loss_and_grad(img, first, st[kind], actions)
            else:
                loss, _ = autograd_loss(pol, img, first, st[kind], actions)
                loss.backward()
            s1.record()
            torch.cuda.synchronize()
        finally:
            for n in names:
                setattr(ops, n, saved[n])
        tot, cnt = collections.defaultdict(float), collections.Counter()
        for n, e0, e1 in rec:
            tot[n] += e0.elapsed_time(e1)
            cnt[n] += 1
        print(f"[{kind}] instrumented fwd+bwd {s0.elapsed_time(s1):.1f} ms; sum of ops {sum(tot.values()):.1f} ms")
        for n, t in sorted(tot.items(), key=lambda kv: -kv[1])[:12]:
            print(f"  {t:8.2f} ms  n={cnt[n]:4d}  {n}")


def kernel_bench(N=2048, width=8762, iters=50):
    """log_softmax_bwd over the two heads' columns of N frames: reads logp and g (8 B per element), writes 2 B."""
    g = torch.Generator(device="cuda").manual_seed(1)
    logp = torch.log_softmax(torch.randn(N, width, device="cuda", generator=g), -1)
    up = torch.randn(N, width, device="cuda", generator=g)
    out = torch.empty(N, (width + 7) // 8 * 8, dtype=torch.bfloat16, device="cuda")

    def run():
        ops.log_softmax_bwd(logp[:, :121], up[:, :121], 0.5, out, 0)
        ops.log_softmax_bwd(logp[:, 121:], up[:, 121:], 0.5, out, 121)

    for _ in range(5):
        run()
    e0, e1 = ev(), ev()
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    nbytes = N * width * 10
    bound = nbytes / 3.35e12 * 1e3
    print(f"log_softmax_bwd N={N} x {width} columns (121 + 8641): {ms * 1e3:.1f} us, {nbytes / ms / 1e9:.2f} TB/s; "
          f"HBM bound at 3.35 TB/s {bound * 1e3:.1f} us ({100 * bound / ms:.0f} % of it)")


def fit(width, B):
    """One autograd step at `width` (and one BCTrainer step for comparison): peak memory of each."""
    torch.cuda.empty_cache()
    pol, img, first, actions, opt = setup(width, B)
    res = {}
    for kind in ("bc", "ag"):
        opt.zero_grad()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = ev(), ev()
        e0.record()
        if kind == "bc":
            BCTrainer(pol).loss_and_grad(img, first, pol.initial_state(B), actions)
            gc.collect()
        else:
            pol.set_autograd(True)
            loss, _ = autograd_loss(pol, img, first, pol.initial_state(B), actions)
            loss.backward()
        opt.step()
        e1.record()
        torch.cuda.synchronize()
        res[kind] = (e0.elapsed_time(e1), torch.cuda.max_memory_allocated())
        torch.cuda.empty_cache()
    nat.device_check()
    print(f"{width} B={B} T={T} one step (first call, includes weight layout): BCTrainer {res['bc'][0]:.0f} ms, peak {res['bc'][1] / 2 ** 30:.2f} GiB; "
          f"autograd {res['ag'][0]:.0f} ms, peak {res['ag'][1] / 2 ** 30:.2f} GiB")


if __name__ == "__main__":
    main()
