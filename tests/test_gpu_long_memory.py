"""Policies with a KV memory longer than 128 frames on the H100, against the reference (tests/golden/long_memory.pt, made by
tools/make_long_memory_golden.py): maxlen 1920 (attention_memory_size 2048, the reference's default) and maxlen 300 at the SMALL config.
The bf16 and fp32 forwards, `loss.backward()` over a two-chunk window with the state attached, BCTrainer and RLTrainer (kl_coef = 0) from
a full memory; the window's gradients also against autograd through the BPTT forced replica; sampled actions of `act` and `GraphedAct`;
`recompute_frames` and a frozen CNN; and the released 128-frame memory loaded into a 1920-frame policy through `resize_memory`."""
import os
import sys

import pytest
import torch

import vpt_b200
from common import make_policy, small_kwargs
from test_autograd_golden import _policy
from test_bptt import window_vs_forced
from test_gpu_rl_training import no_tf32
from video_pre_training_b200 import _native as nat
from video_pre_training_b200.training import BCTrainer, RLTrainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden as MG  # noqa: E402
import make_long_memory_golden as MLG  # noqa: E402

pytestmark = pytest.mark.gpu
# Against the reference the two bf16 forwards round differently, so ReLU / max-pool masks flip and the peaked attention of the perturbed
# weights moves (tests/test_gpu_bptt.py measured up to 0.30 in the CNN and 0.26 outside it at maxlen 8); here, at maxlen 1920 / 300, up to
# 0.27 outside the CNN (r_layer.bias) and 0.47 in it (H100).  These bounds pin the loss, the None pattern and gross errors; the forced
# replica test pins the gradients at the CUDA forward's operating point to 3e-2.
TOL_REST, TOL_CNN = 0.4, 0.7


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(ROOT, "tests", "golden", "long_memory.pt"), weights_only=False)


def _pol(fx, name):
    f = dict(fx[name], wseed=fx["wseed"], perturbed=fx["perturbed"])
    return _policy(f, fx["wseed"]).cuda()


def _cuda(chunk):
    img, first, actions = chunk[:3]
    return img.cuda(), first.cuda(), {k: v.cuda() for k, v in actions.items()}


def _maxrel(a, b):
    return ((a.float().cpu() - b.float()).abs() / b.float().abs().clamp(min=1e-30)).max().item()


def _rel(a, b):
    return ((a.float().cpu() - b.float()).norm() / b.float().norm().clamp(min=1e-30)).item()


def _warm(pol, name):
    st = pol.initial_state(MLG.B)
    with torch.no_grad():
        for img, first, _ in map(_cuda, MLG.warmup_inputs(name)):
            _, st = pol({"img": img}, first, st)
    return st


def _check_grads(pol, ref, loss, ref_loss, what):
    """loss to 1e-2; per parameter the gradient norm and the fixed samples against the reference's, as rel-L2 of the samples"""
    assert abs(loss - ref_loss.item()) < 1e-2 * abs(ref_loss.item()), (what, loss, ref_loss.item())
    named = dict(pol.named_parameters())
    worst = {}
    for n, r in ref.items():
        g = named[n].grad
        assert (g is None) == (r is None), (what, n)
        if r is None or r["norm"].item() == 0:
            continue
        gflat = g.flatten()
        s = gflat[MG.grad_sample_index(n, gflat.numel())]
        worst[n] = max(abs(gflat.norm().item() - r["norm"].item()) / r["norm"].item(), _rel(s, r["sample"]) * r["sample"].norm().item() / r["norm"].item())
    rest = sorted(((n, e) for n, e in worst.items() if ".cnn." not in n), key=lambda kv: -kv[1])
    cnn = sorted(((n, e) for n, e in worst.items() if ".cnn." in n), key=lambda kv: -kv[1])
    print(what, "worst outside the CNN", rest[:3], "in the CNN", cnn[:2])
    return rest[0][1], cnn[0][1]


@pytest.mark.parametrize("name", list(MLG.CONFIGS))
def test_forward_against_the_reference(fx, name):
    pol = _pol(fx, name)
    maxlen = MLG.CONFIGS[name][0] - MLG.CONFIGS[name][1]
    st = pol.initial_state(MLG.B)
    for img, first, _ in map(_cuda, MLG.forward_inputs(name)):
        (pd, v, _), st = pol({"img": img}, first, st)
    nat.device_check()
    ref = fx[name]["forward"]
    c = ref["chunks"][-1]
    errs = dict(camera=_maxrel(pd["camera"], c["pd"]["camera"]), buttons=_maxrel(pd["buttons"][..., MG.COLS], c["pd"]["buttons"]),
                vpred=_rel(v, c["vpred"]))
    rows = MLG.state_rows(maxlen)
    for l, ((m, (k, vv)), (rm, rk, rv)) in enumerate(zip(st, ref["state"])):
        assert torch.equal(m.cpu(), rm), l
        errs[f"k{l}"], errs[f"v{l}"] = _rel(k[:, rows], rk), _rel(vv[:, rows], rv)
    print(name, {k: f"{e:.2e}" for k, e in errs.items()})
    # tests/test_gpu_policy.py's bounds: log-probs 1e-2 max rel, vpred 5e-2 max abs, KV state 3e-2 rel-L2.  After 17 chunks of carried
    # bf16 state with the perturbed weights (q x 30) the logits sit close to the first bound (measured 9.8e-3 camera, 5.0e-3 buttons,
    # KV state 1.8e-2 at maxlen 1920, H100), so the log-probs are held to it as rel-L2 and to twice it elementwise.
    assert errs["camera"] < 2e-2 and errs["buttons"] < 2e-2
    assert _rel(pd["camera"], c["pd"]["camera"]) < 1e-2 and _rel(pd["buttons"][..., MG.COLS], c["pd"]["buttons"]) < 1e-2
    assert (v.float().cpu() - c["vpred"]).abs().max().item() < 5e-2
    assert all(e < 3e-2 for k, e in errs.items() if k[0] in "kv" and k[1:].isdigit())


@pytest.mark.parametrize("name", list(MLG.CONFIGS))
def test_fp32_forward_against_the_reference(fx, name):
    pol = _pol(fx, name).set_precision("fp32")
    st = pol.initial_state(MLG.B)
    for img, first, _ in map(_cuda, MLG.forward_inputs(name)):
        (pd, v, _), st = pol({"img": img}, first, st)
    nat.device_check()
    c = fx[name]["forward"]["chunks"][-1]
    errs = (_maxrel(pd["camera"], c["pd"]["camera"]), _maxrel(pd["buttons"][..., MG.COLS], c["pd"]["buttons"]), _rel(v, c["vpred"]))
    print(name, "fp32", errs)
    assert max(errs) < 1e-3


@pytest.mark.parametrize("name", list(MLG.CONFIGS))
def test_window_backward_against_the_reference(fx, name):
    pol = _pol(fx, name)
    maxlen = MLG.CONFIGS[name][0] - MLG.CONFIGS[name][1]
    warm = _warm(pol, name)
    pol.set_autograd(True, state_grad=True)
    st = [(m, (k.clone().requires_grad_(True), v.clone().requires_grad_(True))) for m, (k, v) in warm]
    s, loss = st, 0.0
    for img, first, actions in map(_cuda, MLG.window_inputs(name)):
        (pd, _, _), s = pol({"img": img}, first, s)
        loss = loss + MLG.bc_loss(pd, actions)
    loss.backward()
    nat.device_check()
    ref = fx[name]["window"]
    rest, cnn = _check_grads(pol, ref["grads"], loss.item(), ref["loss"], f"{name} window")
    rows = MLG.state_rows(maxlen)
    for l, ((_, (k, v)), r) in enumerate(zip(st, ref["state_grad"])):
        e = (_rel(k.grad[:, rows], r["k"]), _rel(v.grad[:, rows], r["v"]), abs(k.grad.norm().item() / r["norm"][0].item() - 1),
             abs(v.grad.norm().item() / r["norm"][1].item() - 1))
        print(name, "state gradient layer", l, e)
        assert max(e) < 0.3, (l, e)  # measured up to 0.16
    assert rest < TOL_REST and cnn < TOL_CNN


def test_window_backward_against_the_forced_replica(fx):
    """at the CUDA forward's operating point the gradients are pinned as tightly as tests/test_gpu_bptt.py pins them at maxlen 128"""
    import vpt_oracle as O

    name = "m1920"
    pol = _pol(fx, name)
    warm = _warm(pol, name)
    pol.set_autograd(True, state_grad=True)
    sd = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    cfg = O.Cfg(**fx[name]["policy_kwargs"])
    loss, loss_f, worst = window_vs_forced(pol, sd, cfg, list(map(_cuda, MLG.window_inputs(name))), (0, 1), ctx=no_tf32, st=warm)
    nat.device_check()
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("maxlen 1920 window vs BPTT forced replica, worst", top)
    assert abs(loss - loss_f) < 1e-3 * abs(loss_f)
    assert top[0][1] < 3e-2


def test_bc_trainer_against_the_reference(fx):
    pol = _pol(fx, "m1920")
    warm = _warm(pol, "m1920")
    img, first, actions, *_ = MLG.chunk_inputs("m1920")
    loss, _ = BCTrainer(pol).loss_and_grad(img.cuda(), first.cuda(), warm, {k: v.cuda() for k, v in actions.items()})
    nat.device_check()
    rest, cnn = _check_grads(pol, fx["m1920"]["chunk"]["grads"], loss.item(), fx["m1920"]["chunk"]["loss"], "BCTrainer")
    assert rest < TOL_REST and cnn < TOL_CNN


def test_rl_trainer_against_the_reference(fx):
    pol = _pol(fx, "m1920")
    warm = _warm(pol, "m1920")
    img, first, actions, adv, returns, _ = MLG.chunk_inputs("m1920")
    ref = fx["m1920"]["rl"]
    loss, _ = RLTrainer(pol).loss_and_grad(img.cuda(), first.cuda(), warm, {k: v.cuda() for k, v in actions.items()}, ref["old_logprob"].cuda(),
                                           adv.cuda(), returns.cuda(), None, vf_coef=MLG.VF_COEF, kl_coef=0.0, clip=MLG.CLIP)
    nat.device_check()
    rest, cnn = _check_grads(pol, ref["grads"], loss.item(), ref["loss"], "RLTrainer")
    assert rest < TOL_REST and cnn < TOL_CNN


def test_loop_against_the_reference(fx):
    pol = _pol(fx, "m1920")
    warm = _warm(pol, "m1920")
    pol.set_autograd(True, state_grad=True)
    st, loss = warm, 0.0
    for img, first, actions in map(_cuda, MLG.loop_inputs("m1920")):
        (pd, _, _), st = pol({"img": img}, first, st)
        loss = loss + MLG.bc_loss(pd, actions) / MLG.LOOP_CALLS
    loss.backward()
    nat.device_check()
    rest, cnn = _check_grads(pol, fx["m1920"]["loop"]["grads"], loss.item(), fx["m1920"]["loop"]["loss"], "loop")
    assert rest < TOL_REST and cnn < TOL_CNN


@pytest.mark.parametrize("B", [1, 3])
def test_act_and_graphed_act_sample_the_same_actions(fx, B):
    pol = _pol(fx, "m1920")
    g = torch.Generator().manual_seed(3)
    frames = torch.randint(0, 256, (6, B, 32, 32, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(B, dtype=torch.bool, device="cuda")
    ga = vpt_b200.policy.GraphedAct(pol, B)
    outs = []
    for fn in (pol.act, ga):
        torch.manual_seed(11)
        st, acts = pol.initial_state(B), []
        for f in frames:
            ac, st, _ = fn({"img": f}, first, st)
            acts.append({k: v.clone() for k, v in ac.items()})
        outs.append(acts)
    nat.device_check()
    for a, b in zip(*outs):
        for k in a:
            assert torch.equal(a[k], b[k]), k


def _bc_grads(pol, trainer, img, first, st, actions):
    pol.zero_grad(set_to_none=True)
    loss, _ = trainer.loss_and_grad(img, first, st, actions)
    return loss.item(), {n: p.grad.clone() for n, p in pol.named_parameters() if p.grad is not None}


def test_recompute_and_frozen_cnn_keep_the_gradients_at_maxlen_1920(fx):
    pol = _pol(fx, "m1920")
    warm = _warm(pol, "m1920")
    img, first, actions = _cuda(MLG.chunk_inputs("m1920"))
    l0, g0 = _bc_grads(pol, BCTrainer(pol), img, first, warm, actions)
    l1, g1 = _bc_grads(pol, BCTrainer(pol, recompute_frames=256), img, first, warm, actions)
    assert l1 == l0 and set(g1) == set(g0) and all(torch.equal(g1[n], g0[n]) for n in g0)
    for n, p in pol.named_parameters():
        if n.startswith("net.img_process.cnn"):
            p.requires_grad_(False)
    l2, g2 = _bc_grads(pol, BCTrainer(pol), img, first, warm, actions)
    nat.device_check()
    assert l2 == l0 and g2 and all(torch.equal(g2[n], g0[n]) for n in g2)
    assert not any(n.startswith("net.img_process.cnn") for n in g2)


def test_resize_memory_loads_the_128_frame_weights():
    """a first chunk from initial_state sees no memory beyond itself, so 128 and 1920 frames of memory give the same outputs"""
    pol128, sd, _ = make_policy(small_kwargs(timesteps=128, attention_memory_size=256))
    kw = small_kwargs(timesteps=128, attention_memory_size=2048)
    pol1920 = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
    pol1920.load_state_dict(vpt_b200.resize_memory(sd, 1920))
    g = torch.Generator().manual_seed(4)
    img = torch.randint(0, 256, (2, 128, 32, 32, 3), dtype=torch.uint8, generator=g).cuda()
    first = torch.zeros(2, 128, dtype=torch.bool, device="cuda")
    outs = []
    for pol in (pol128.cuda(), pol1920.cuda()):
        (pd, v, _), _ = pol({"img": img}, first, pol.initial_state(2))
        outs.append((pd, v))
    nat.device_check()
    (pa, va), (pb, vb) = outs
    for k in pa:
        assert _maxrel(pb[k], pa[k].cpu()) < 1e-2, k
    assert _rel(vb, va.cpu()) < 1e-2
