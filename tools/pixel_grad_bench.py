#!/usr/bin/env python
"""Float frames and the image gradient: ms per call, peak memory, and the two image-gradient kernels against their HBM bounds.

    python tools/pixel_grad_bench.py [--steps 3] [--warmup 1]

    fwd2x      the 2x inference forward at B x T = 128 x 128 with fp32 frames against uint8 frames holding the same values (outputs
               compared bit for bit)
    sal2x      the 2x saliency step at B = 16, T = 128: every parameter frozen, the camera-head loss, `loss.backward()` to the pixels;
               beside the all-trainable `loss.backward()` step of the BC loss on uint8 frames
    idm4x      the same for the 4x IDM at B = 4, T = 128 (the camera-head loss for both)
    kernels    vpt_firstconv_dimg at 2x (C0 = 128, 2048 frames) and vpt_conv3d_t5_dimg at 4x (C = 128, 512 frames): CUDA events over 20
               launches, against the bytes each must move (from the shapes) at the data-sheet 3.35 TB/s

Times are CUDA events around the whole call (medians over the timed calls, the variants alternating); peak memory is
`max_memory_allocated` reset before each timed call.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200
from video_pre_training_b200 import ops

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--out", default=None, help="also write the results as JSON here")
a = ap.parse_args()
ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
GiB = 2 ** 30
HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn):
    """-> (ms, peak GiB, result) of one call."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = ev(), ev()
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), torch.cuda.max_memory_allocated() / GiB, r


def alternate(variants):
    """{name: fn} run in turn, warm-up then timed -> {name: (median ms, max peak GiB, last result)}."""
    res = {k: [] for k in variants}
    last = {}
    for i in range(a.warmup + a.steps):
        for k, fn in variants.items():
            ms, peak, r = timed(fn)
            last[k] = r
            if i >= a.warmup:
                res[k].append((ms, peak))
    return {k: (sorted(m for m, _ in v)[len(v) // 2], max(p for _, p in v), last[k]) for k, v in res.items()}


def agent(width):
    torch.manual_seed(0)
    return vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(width), vpt_b200.PI_HEAD_KWARGS).cuda()


def camera_loss(pd):
    return -pd["camera"][..., 0, :7].sum() / pd["camera"].numel()


def main():
    name, power = card()
    out = dict(card=name, power_limit=power)
    g = torch.Generator().manual_seed(0)
    # ---- fwd2x
    pol = agent("2x")
    B, T = 128, 128
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    imgf = img.float()
    first = torch.zeros(B, T, dtype=torch.bool).cuda()
    st = pol.initial_state(B)

    def fwd(x):
        with torch.no_grad():
            (pd, v, _), _ = pol({"img": x}, first, st)
        return pd, v
    r = alternate({"u8": lambda: fwd(img), "f32": lambda: fwd(imgf)})
    same = torch.equal(r["u8"][2][1], r["f32"][2][1]) and all(torch.equal(r["u8"][2][0][k], r["f32"][2][0][k]) for k in r["u8"][2][0])
    out["fwd2x"] = dict(u8_ms=r["u8"][0], f32_ms=r["f32"][0], bit_identical=same)
    print(f"2x forward B x T = 128 x 128: uint8 {r['u8'][0]:.1f} ms, fp32 frames {r['f32'][0]:.1f} ms, outputs bit-identical: {same}")
    del img, imgf, r, st
    # ---- sal2x
    B = 16
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool).cuda()
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g).cuda(), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g).cuda()}
    frozen = agent("2x").set_autograd(True)
    for p in frozen.parameters():
        p.requires_grad_(False)
    pol.set_autograd(True)
    x = (img.float() + torch.rand(img.shape, device="cuda")).requires_grad_(True)

    def saliency():
        x.grad = None
        (pd, _, _), _ = frozen({"img": x}, first, frozen.initial_state(B))
        camera_loss(pd).backward()

    def train():
        for p in pol.parameters():
            p.grad = None
        (pd, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
        (-pol.logprob(actions, pd).mean()).backward()
    r = alternate({"saliency": saliency, "trainable": train})
    out["sal2x"] = {k: dict(ms=v[0], peak_gib=v[1]) for k, v in r.items()}
    print(f"2x B = 16, T = 128: saliency (all frozen, img.grad) {r['saliency'][0]:.1f} ms, peak {r['saliency'][1]:.1f} GiB; "
          f"all-trainable loss.backward() {r['trainable'][0]:.1f} ms, peak {r['trainable'][1]:.1f} GiB")
    del pol, frozen, x, img, r
    # ---- idm4x
    torch.manual_seed(0)
    mk = lambda: vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs()).cuda()  # noqa: E731
    idm, idm_f = mk().set_autograd(True), mk().set_autograd(True)
    for p in idm_f.parameters():
        p.requires_grad_(False)
    B = 4
    img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, T, dtype=torch.bool).cuda()
    x = (img.float() + torch.rand(img.shape, device="cuda")).requires_grad_(True)

    def idm_saliency():
        x.grad = None
        (pd, _, _), _ = idm_f({"img": x}, first, idm_f.initial_state(B))
        camera_loss(pd).backward()

    def idm_train():
        for p in idm.parameters():
            p.grad = None
        (pd, _, _), _ = idm({"img": img}, first, idm.initial_state(B))
        camera_loss(pd).backward()
    r = alternate({"saliency": idm_saliency, "trainable": idm_train})
    out["idm4x"] = {k: dict(ms=v[0], peak_gib=v[1]) for k, v in r.items()}
    print(f"4x IDM B = 4, T = 128: saliency {r['saliency'][0]:.1f} ms, peak {r['saliency'][1]:.1f} GiB; "
          f"all-trainable loss.backward() {r['trainable'][0]:.1f} ms, peak {r['trainable'][1]:.1f} GiB")
    del idm, idm_f, x, img, r
    # ---- kernels
    F_, C0 = 2048, 128
    frames = torch.rand((F_, 128, 128, 3), device="cuda") * 255
    w, b = torch.randn((C0, 27), device="cuda") / 255, torch.randn((C0,), device="cuda") * 0.1
    dy = torch.randn((F_, 65, 65, C0), device="cuda").to(torch.bfloat16)
    c3 = torch.randn((512, 129, 129, 128), device="cuda").to(torch.bfloat16)
    w3 = torch.randn((128, 15), device="cuda") / 255
    kern = {
        "firstconv_dimg 2x, 2048 frames": (lambda: ops.firstconv_dimg(frames, w, b, dy, C0), dy.numel() * 2 + frames.numel() * 4 * 2),
        "conv3d_t5_dimg 4x, 512 frames": (lambda: ops.conv3d_t5_dimg(c3, w3, 4, 128, 128, 128), c3.numel() * 2 + 512 * 128 * 128 * 3 * 4),
    }
    out["kernels"] = {}
    for k, (fn, nbytes) in kern.items():
        for _ in range(3):
            fn()
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(20):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        bound = nbytes / HBM * 1e3
        out["kernels"][k] = dict(ms=ms, hbm_bound_ms=bound, gbytes=nbytes / 1e9)
        print(f"{k}: {ms:.2f} ms, HBM bound {bound:.2f} ms ({nbytes / 1e9:.2f} GB at 3.35 TB/s): {bound / ms * 100:.0f} % of it")
    print(f"card: {name}, power limit {power}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


main()
