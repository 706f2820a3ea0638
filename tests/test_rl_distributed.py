"""CPU, gloo, world size 2: the RL fine-tuning step data-parallel (mirrors test_idm_distributed.py).  Sequences are sharded across ranks, the
weights are replicated, and the flat gradient bucket is all-reduced once, or in two parts with the upper slice reduced while the CNN
backward still runs.  Both must equal the gradient of the whole batch computed in one process, and every rank must end with the EWMA
normaliser that one process computes on the global batch."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_distributed import ROOT, _free_port


def _rl_worker(rank, world, port, q):
    for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import emu_rl_ops
    import vpt_oracle as O
    from common import emulation
    from test_rl_training import NORM, make_pair, make_rl_batch, ref_pd
    from video_pre_training_b200 import ops, parallel
    from video_pre_training_b200.training import RLTrainer

    pol, sd, sd_ref, cfg = make_pair()  # identical replicas
    nz = pol.value_head.normalizer
    norm0 = {k: getattr(nz, k).detach().clone() for k in NORM}
    B, T = 4, 8
    g = torch.Generator().manual_seed(0)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    pd_ref, _ = ref_pd(cfg, sd_ref, img, first, O.initial_state(cfg, B))
    with torch.no_grad():
        (pd0, _, _), _ = O.agent_policy_forward(sd, cfg, img, first, O.initial_state(cfg, B))
    old, adv, returns = make_rl_batch(g, O.logprob(pd0, actions), B, T)
    params = [p for p in pol.parameters() if p.requires_grad]
    opt = parallel.FlatAdamDP(params, lr=1e-3)
    split = opt.offset_of(pol.net.img_process.cnn.dense.norm.weight)
    below = {id(p) for p in params if opt.offset_of(p) < split}
    names_below = [n for n, p in pol.named_parameters() if id(p) in below]
    # what is still to come when upper_grads_ready fires is exactly the slice below the split (the value head is above it)
    assert names_below and all(n.startswith("net.img_process.cnn.stacks.") for n in names_below), names_below
    assert opt.offset_of(pol.value_head.linear.weight) > split
    lo, hi = parallel.shard_range(B, rank, world)

    def reset_norm():
        with torch.no_grad():
            for k in NORM:
                getattr(nz, k).copy_(norm0[k])

    kwargs = dict(vf_coef=0.5, kl_coef=0.1)
    with emulation():
        for n in ("ppo_coef", "rl_head_bwd", "ewma_sums", "value_bwd"):
            setattr(ops, n, getattr(emu_rl_ops, n))
        sl = lambda x: x[lo:hi]
        shard = (sl(img), sl(first), pol.initial_state(hi - lo), {k: sl(v) for k, v in actions.items()}, sl(old), sl(adv), sl(returns),
                 {k: sl(v) for k, v in pd_ref.items()})
        opt.zero_grad()
        RLTrainer(pol).loss_and_grad(*shard, **kwargs)
        w = opt.reduce_gradients()
        dp_grad = opt.flat_g.clone() / w
        dp_norm = torch.stack([getattr(nz, k).detach().reshape(()).clone() for k in NORM])
        reset_norm()
        opt.zero_grad()
        RLTrainer(pol).loss_and_grad(*shard, upper_grads_ready=lambda: opt.reduce_async(split, opt.n), **kwargs)
        assert opt._pending is not None
        opt.reduce_gradients()
        assert opt._pending is None and torch.equal(opt.flat_g / w, dp_grad)
        gathered = [torch.empty_like(dp_norm) for _ in range(world)]
        dist.all_gather(gathered, dp_norm)
        same_on_ranks = all(torch.equal(x, gathered[0]) for x in gathered)
        dist.destroy_process_group()  # the single-process reference below must not all-reduce
        if rank == 0:  # the same global batch in one process
            reset_norm()
            opt.zero_grad()
            RLTrainer(pol).loss_and_grad(img, first, pol.initial_state(B), actions, old, adv, returns, pd_ref, **kwargs)
            err = ((dp_grad - opt.flat_g).norm() / opt.flat_g.norm()).item()
            ov = opt.offset_of(pol.value_head.linear.weight)
            nv = pol.value_head.linear.weight.numel()
            err_v = ((dp_grad[ov:ov + nv] - opt.flat_g[ov:ov + nv]).norm() / opt.flat_g[ov:ov + nv].norm()).item()
            single = torch.stack([getattr(nz, k).detach().reshape(()).clone() for k in NORM])
            q.put((rank, w, err, err_v, same_on_ranks, bool(torch.allclose(dp_norm, single, rtol=1e-6, atol=0))))
        else:
            q.put((rank, w, 0.0, 0.0, same_on_ranks, True))


def test_rl_data_parallel_gradients_and_normaliser_equal_the_global_batch_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_rl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=600) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(w == 2 for _, w, _, _, _, _ in res)
    assert all(r[4] and r[5] for r in res), res
    assert res[0][2] < 2e-2 and res[0][3] < 2e-2, res
