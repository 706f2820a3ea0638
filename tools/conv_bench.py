#!/usr/bin/env python
"""Kernel timing of vpt_conv3x3_zp at the four convolution shape classes of the 2x policy forward (frames in chunks of F = 2048).

Every class runs the launches the forward makes at that shape, with the same arguments (per-frame GroupNorm fold `mr` + `S1/S2`,
block 0's two-norm composition `Ef` / `res_scale, res_shift`, the residual on each block's second conv, statistics partials where
the forward asks for them), and is timed with CUDA events around the kernel launches only (no statistics finalize).  Each class is
timed with the epilogue on and with the epilogue body switched off (vpt_set_conv_pair_mode(0x20): the main loop only; the
accumulators are dropped), so the gap is what the epilogue costs.
    python tools/conv_bench.py [--frames 2048] [--reps 3] [--json OUT]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import vpt_b200  # noqa: E402,F401
from video_pre_training_b200 import _native as nat  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16

# (name, H = W, Cin, Cout, launch pattern); patterns: "block0" = Ef conv + res_scale/res_shift residual conv (inference fold of the
# post-pool norm), "block" = plain conv + residual conv, "first" = a stack's first conv (no statistics)
CLASSES = [
    ("64x64 128->128 (stack 0 blocks)", 64, 128, 128, ["block0", "block"]),
    ("64x64 128->256 (stack 1 first conv)", 64, 128, 256, ["first"]),
    ("32x32 256->256 (stack 1 blocks + stack 2 first conv)", 32, 256, 256, ["block0", "block", "first"]),
    ("16x16 256->256 (stack 2 blocks)", 16, 256, 256, ["block0", "block"]),
]


def zp_rand(F_, H, W, C_, dev):
    t = torch.randn(F_, H + 1, W + 1, C_, device=dev).to(torch.bfloat16)
    t[:, H] = 0
    t[:, :, W] = 0
    return t


def launch(l, x, Wb, H, W, out, part, mr=None, S1=None, S2=None, residual=None, Ef=None, rs=None, rb=None):
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    a = nat.ConvZpArgs()
    a.x, a.w, a.F, a.H, a.W, a.Cin, a.Cout = p(x), p(Wb), x.shape[0], H, W, x.shape[3], Wb.shape[0]
    a.mr, a.S1, a.S2, a.relu, a.residual, a.out, a.stat_part = p(mr), p(S1), p(S2), 1, p(residual), p(out), p(part)
    a.Ef, a.res_scale, a.res_shift = p(Ef), p(rs), p(rb)
    nat.check(l.vpt_conv3x3_zp(C.byref(a), torch.cuda.current_stream().cuda_stream), "vpt_conv3x3_zp")


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit, sm_clock, max_sm_clock"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia-smi"] = f"unavailable ({e})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "conv_bench needs a GPU"
    dev = torch.device("cuda", 0)
    l = nat.lib()
    F_ = a.frames
    torch.manual_seed(0)
    rows = []
    for name, HW, Cin, N, pattern in CLASSES:
        H = W = HW
        FS = (H + 1) * (W + 1)
        P = l.vpt_conv_zp_stat_parts(F_, H, W, N)
        x = zp_rand(F_, H, W, Cin, dev)
        res = zp_rand(F_, H, W, N, dev) if N == Cin else None
        Wb = (torch.randn(N, 9 * Cin, device=dev) * (9 * Cin) ** -0.5).to(torch.bfloat16)
        Wb2 = (torch.randn(N, 9 * N, device=dev) * (9 * N) ** -0.5).to(torch.bfloat16)
        mr = torch.stack([torch.randn(F_, device=dev) * 0.1, torch.rand(F_, device=dev) + 0.5], 1).contiguous()
        mrE = torch.stack([torch.zeros(F_, device=dev), torch.rand(F_, device=dev) + 0.5], 1).contiguous()
        S1, S2 = torch.randn(9, N, device=dev), torch.randn(9, N, device=dev)
        Ef = torch.randn(F_, 9, N, device=dev)
        rs, rb = torch.rand(F_, N, device=dev) + 0.5, torch.randn(F_, N, device=dev) * 0.1
        out = torch.empty(F_, H + 1, W + 1, N, dtype=torch.bfloat16, device=dev)
        part = torch.empty(F_ * FS, P, 2, dtype=torch.float32, device=dev)
        calls = []
        for pat in pattern:
            if pat == "first":
                calls.append(lambda: launch(l, x, Wb, H, W, out, None, mr=mr, S1=S1, S2=S2))
            elif pat == "block0":
                calls.append(lambda: launch(l, x, Wb, H, W, out, part, mr=mrE, Ef=Ef))
                calls.append(lambda: launch(l, x, Wb2, H, W, out, part, mr=mr, S1=S1, S2=S2, residual=res, rs=rs, rb=rb))
            else:
                calls.append(lambda: launch(l, x, Wb, H, W, out, part, mr=mr, S1=S1, S2=S2))
                calls.append(lambda: launch(l, x, Wb2, H, W, out, part, mr=mr, S1=S1, S2=S2, residual=res))
        alg = 2.0 * F_ * H * W * N * 9 * Cin
        zp = 2.0 * ((F_ * FS + 127) // 128 * 128) * N * 9 * Cin  # rows the kernel computes: whole 128-row tiles of the ZP layout
        row = dict(cls=name, launches=len(calls))
        for tag, mode in (("epi_on", 0), ("epi_off", 0x20)):
            l.vpt_set_conv_pair_mode(mode)
            for c in calls:
                c()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                for c in calls:
                    c()
            e1.record()
            torch.cuda.synchronize()
            nat.device_check()
            ms = e0.elapsed_time(e1) / (a.reps * len(calls))
            row[tag] = dict(ms=ms, alg_tflops=alg / ms / 1e9, zp_tflops=zp / ms / 1e9, zp_share_of_peak=zp / ms / 1e9 / PEAK_TFLOPS)
        l.vpt_set_conv_pair_mode(0)
        rows.append(row)
        del x, res, out, part
        torch.cuda.empty_cache()
    info = card_info()
    print(f"card: {info}")
    print(f"F = {F_}; ms per launch; TFLOP/s algorithmic (H*W pixels) / over the ZP rows computed; epilogue off = pair mode 0x20")
    print(f"{'class':55s} {'n':>2s} | {'ms':>7s} {'alg':>6s} {'zp':>6s} {'%pk':>5s} | {'ms off':>7s} {'alg':>6s} {'zp':>6s} {'%pk':>5s}")
    for r in rows:
        on, off = r["epi_on"], r["epi_off"]
        print(f"{r['cls']:55s} {r['launches']:2d} | {on['ms']:7.3f} {on['alg_tflops']:6.0f} {on['zp_tflops']:6.0f} {100 * on['zp_share_of_peak']:5.1f}"
              f" | {off['ms']:7.3f} {off['alg_tflops']:6.0f} {off['zp_tflops']:6.0f} {100 * off['zp_share_of_peak']:5.1f}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=info, frames=F_, classes=rows), f, indent=1)


if __name__ == "__main__":
    main()
