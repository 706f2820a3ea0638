#!/usr/bin/env python
"""Device memory that stays allocated when three training paths run on one policy: a 2x policy, one BCTrainer call, one RLTrainer call
and one `loss.backward()` through the differentiable forward (`set_autograd`), then `torch.cuda.memory_allocated()` with every `.grad`
dropped: the parameters, the kernel-layout weight copies and whatever the trainers keep between calls.  Also prints, from the shapes,
the size of one bf16 copy of the weight matrices (what one extra set of backward layouts costs), and the card and its power limit from
the same run.

    python tools/layout_memory.py [--B 2] [--T 16]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vpt_b200

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=2)
ap.add_argument("--T", type=int, default=16)
a = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
print(f"card: {q.stdout.strip() or torch.cuda.get_device_name()}  (name, power limit)")
torch.manual_seed(0)
pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs("2x"), vpt_b200.PI_HEAD_KWARGS).cuda()
B, T = a.B, a.T
g = torch.Generator(device="cuda").manual_seed(0)
img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g),
           "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
old = -14.0 + 0.1 * torch.randn(B, T, device="cuda", generator=g)
adv, returns = torch.randn(B, T, device="cuda", generator=g), 3.0 + torch.randn(B, T, device="cuda", generator=g)

bc, rl = vpt_b200.BCTrainer(pol), vpt_b200.RLTrainer(pol)
bc.loss_and_grad(img, first, pol.initial_state(B), actions)
rl.loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, vf_coef=0.5, kl_coef=0.0)
(pd, _, _), _ = pol.set_autograd(True)({"img": img}, first, pol.initial_state(B))
(-pol.logprob(actions, pd).mean()).backward()
del pd
for p in pol.parameters():
    p.grad = None
torch.cuda.synchronize()
params = sum(p.numel() * p.element_size() for p in pol.parameters())
matrices = sum(p.numel() * 2 for p in pol.parameters() if p.dim() >= 2)
print(f"after one BC call, one RL call and one differentiable-forward backward on one 2x policy (B={B}, T={T}): "
      f"memory_allocated {torch.cuda.memory_allocated() / 2 ** 30:.3f} GiB; parameters {params / 2 ** 30:.3f} GiB; "
      f"one bf16 copy of the weight matrices (from the shapes) {matrices / 2 ** 30:.3f} GiB")
