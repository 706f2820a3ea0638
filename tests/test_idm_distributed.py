"""CPU, gloo, world size 2: the IDM training step data-parallel (mirrors test_distributed.py's BC test).  Sequences are sharded across
ranks, the weights are replicated, and the flat gradient bucket is all-reduced once, or in two parts with the upper slice reduced while
the CNN backward still runs.  Both must equal the gradient of the whole batch computed in one process."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_distributed import ROOT, _free_port


def _idm_worker(rank, world, port, q):
    for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import emu_idm_ops
    from common import emulation
    from test_idm_training import make_batch, make_idm
    from video_pre_training_b200 import ops, parallel
    from video_pre_training_b200.training import IDMTrainer

    pol, _, _ = make_idm(seed=0)  # identical replicas
    B, T = 4, 8
    img, first, actions = make_batch(torch.Generator().manual_seed(0), B=B, T=T)
    params = IDMTrainer.optimizer_params(pol)
    opt = parallel.FlatAdamDP(params, lr=1e-3)
    split = opt.offset_of(pol.net.img_process.cnn.dense.norm.weight)
    below = {id(p) for p in params if p.numel() > 0 and opt.offset_of(p) < split}  # (an empty parameter has no slice)
    names_below = [n for n, p in pol.named_parameters() if id(p) in below]
    # what is still to come when upper_grads_ready fires is exactly the slice below the split
    assert names_below and all(n.startswith(("net.conv3d_layer.", "net.img_process.cnn.stacks.")) for n in names_below), names_below
    lo, hi = parallel.shard_range(B, rank, world)
    with emulation():
        for n in ("conv3d_t5_bwd", "softmax_nll_bwd_grouped"):
            setattr(ops, n, getattr(emu_idm_ops, n))
        opt.zero_grad()
        shard = (img[lo:hi], first[lo:hi], pol.initial_state(hi - lo), {k: v[lo:hi] for k, v in actions.items()})
        IDMTrainer(pol).loss_and_grad(*shard)
        w = opt.reduce_gradients()
        dp_grad = opt.flat_g.clone() / w
        opt.zero_grad()
        IDMTrainer(pol).loss_and_grad(*shard, upper_grads_ready=lambda: opt.reduce_async(split, opt.n))
        assert opt._pending is not None
        opt.reduce_gradients()
        assert opt._pending is None and torch.equal(opt.flat_g / w, dp_grad)
        if rank == 0:  # the same global batch in one process
            opt.zero_grad()
            IDMTrainer(pol).loss_and_grad(img, first, pol.initial_state(B), actions)
            err = ((dp_grad - opt.flat_g).norm() / opt.flat_g.norm()).item()
            o3 = opt.offset_of(pol.net.conv3d_layer.layer.weight)
            n3 = pol.net.conv3d_layer.layer.weight.numel()
            err3 = ((dp_grad[o3:o3 + n3] - opt.flat_g[o3:o3 + n3]).norm() / opt.flat_g[o3:o3 + n3].norm()).item()
            q.put((rank, w, err, err3))
        else:
            q.put((rank, w, 0.0, 0.0))
    dist.destroy_process_group()


def test_idm_data_parallel_gradients_equal_the_global_batch_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_idm_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=600) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(w == 2 for _, w, _, _ in res)
    assert res[0][2] < 2e-2 and res[0][3] < 2e-2, res
