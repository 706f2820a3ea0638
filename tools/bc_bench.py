#!/usr/bin/env python
"""BC fine-tune step (BASELINE configs[3]: 3x width, bf16, B=16 clips per GPU, T=128, data-parallel): forward with tape +
hand-written backward + ONE NCCL all-reduce over the flat gradient bucket + ONE fused Adam launch per step.

    python tools/bc_bench.py [--width 3x] [--batch 16] [--steps 3]
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/bc_bench.py ...      (weak scaling)

Prints ms/step (max over ranks, CUDA events), frames/s and the split forward / backward / reduce+Adam."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import vpt_b200
from video_pre_training_b200 import _native as nat, ops
from video_pre_training_b200.parallel import FlatAdamDP
from video_pre_training_b200.training import BCTrainer

ap = argparse.ArgumentParser()
ap.add_argument("--width", default="3x")
ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--profile", action="store_true", help="per-GEMM timing of one step (tensor-core kernels only)")
ap.add_argument("--no-overlap", action="store_true", help="one all-reduce after the backward instead of overlapping the upper slice")
ap.add_argument("--ops", action="store_true", help="per-op CUDA-event breakdown of one step (outer ops include the ops they call)")
a = ap.parse_args()
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
torch.manual_seed(0)
pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), vpt_b200.policy_kwargs(a.width), vpt_b200.PI_HEAD_KWARGS).cuda()
B, T = a.batch, 128
g = torch.Generator(device="cuda").manual_seed(rank)
img = torch.randint(0, 256, (B, T, 128, 128, 3), dtype=torch.uint8, device="cuda", generator=g)
first = torch.zeros(B, T, dtype=torch.bool, device="cuda")
actions = {"camera": torch.randint(0, 121, (B, T, 1), device="cuda", generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), device="cuda", generator=g)}
tr = BCTrainer(pol)
opt = FlatAdamDP([p for n, p in pol.named_parameters() if not n.startswith("value_head")], lr=0.000181, weight_decay=0.039428)  # behavioural_cloning.py:38-39
state = pol.initial_state(B)
# everything from the dense layer on (98 % of the bucket) is final before the ImpalaCNN backward starts
split = opt.offset_of(pol.net.img_process.cnn.dense.norm.weight)
hook = None if a.no_overlap else (lambda: opt.reduce_async(split, opt.n))
ev = lambda: torch.cuda.Event(enable_timing=True)


def step(timed=None):
    global state
    opt.zero_grad()
    if timed:
        timed[0].record()
    loss, state = tr.loss_and_grad(img, first, state, actions, upper_grads_ready=hook)
    if timed:
        timed[1].record()
    opt.step()
    if timed:
        timed[2].record()
    return loss


losses = []
for _ in range(a.warmup):
    losses.append(step().item())
torch.cuda.synchronize()
nat.device_check()
if world > 1:
    dist.barrier()
l0 = ops.LAUNCHES
marks = [(ev(), ev(), ev()) for _ in range(a.steps)]
for i in range(a.steps):
    losses.append(step(marks[i]))
torch.cuda.synchronize()
launches = (ops.LAUNCHES - l0) // a.steps
fb = sum(m[0].elapsed_time(m[1]) for m in marks) / a.steps
ad = sum(m[1].elapsed_time(m[2]) for m in marks) / a.steps
tot = torch.tensor([marks[0][0].elapsed_time(marks[-1][2]) / a.steps], device="cuda")
if world > 1:
    dist.all_reduce(tot, op=dist.ReduceOp.MAX)
if rank == 0:
    nparam = sum(p.numel() for p in pol.parameters())
    ms = tot.item()
    print(f"BC step {a.width} B={B}/gpu T={T} x{world} GPU: {ms:.1f} ms/step, {world*B*T/ms*1000:.0f} frames/s; fwd+bwd {fb:.1f} ms, "
          f"all-reduce+Adam {ad:.1f} ms; {launches} launches/step; params {nparam/1e6:.1f} M; peak mem {torch.cuda.max_memory_allocated()/2**30:.1f} GiB; "
          f"loss {float(losses[0]):.4f} -> {float(losses[-1]):.4f}")
if a.profile and rank == 0:
    ops.GEMM_PROFILE = []
    step()
    torch.cuda.synchronize()
    agg = {}
    for e0, e1, fl, tag, shape in ops.GEMM_PROFILE:
        k = (tag, shape)
        t, f, n = agg.get(k, (0.0, 0.0, 0))
        agg[k] = (t + e0.elapsed_time(e1), f + fl, n + 1)
    ops.GEMM_PROFILE = None
    tt = sum(v[0] for v in agg.values())
    print(f"tensor-core kernels: {tt:.1f} ms of the step")
    for (tag, shape), (t, f, n) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:24]:
        print(f"  {t:8.2f} ms  n={n:3d}  {tag:7s} {str(shape):28s} {f/t/1e9:7.0f} TFLOP/s")
if a.ops and rank == 0:
    import collections
    names = ["gemm", "conv3x3_zp", "wgrad", "firstconv_pool", "maxpool3s2", "affine_norm", "affine_norm_zp", "add_zp", "attention", "relu_mask",
             "group_sums", "col_sums", "norm_sums", "norm_bwd_apply", "maxpool3s2_bwd", "firstconv_bwd", "attention_bwd", "softmax_bwd", "copy_rows",
             "log_softmax", "gather_logprob", "stats_finalize"]
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
        setattr(ops, n, wrap(n, getattr(ops, n)))
    s0, s1, s2 = ev(), ev(), ev()
    opt.zero_grad()
    s0.record()
    loss, state = tr.loss_and_grad(img, first, state, actions)
    s1.record()
    opt.step()
    s2.record()
    torch.cuda.synchronize()
    tot, cnt = collections.defaultdict(float), collections.Counter()
    for n, e0, e1 in rec:
        tot[n] += e0.elapsed_time(e1)
        cnt[n] += 1
    p0, p1, p2 = ev(), ev(), ev()   # weight re-layout (every parameter changed in opt.step): forward folds, backward transposes
    p0.record()
    pol.net.prepared(); pol._heads_prepared()
    p1.record()
    pol.net.prepared_backward(); pol._heads_prepared_backward(tr._head_layers())
    p2.record()
    torch.cuda.synchronize()
    print(f"instrumented step: fwd+bwd {s0.elapsed_time(s1):.1f} ms, adam {s1.elapsed_time(s2):.1f} ms; sum of ops {sum(tot.values()):.1f} ms; "
          f"weight re-layout after the step: forward {p0.elapsed_time(p1):.1f} ms + backward {p1.elapsed_time(p2):.1f} ms")
    for n, t in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"  {t:8.2f} ms  n={cnt[n]:4d}  {n}")
if world > 1:
    dist.destroy_process_group()
