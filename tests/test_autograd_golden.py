"""The differentiable forward against the reference's own autograd (tests/golden/autograd_gradient.pt, made by
tools/make_autograd_golden.py): the inner loop of behavioural_cloning.py:86-123 as written (one frame per call, two episodes, state
carried and detached, backward per sample) and a camera-only custom loss.  Live where the reference checkout is present (the stored
fixture is then also re-derived and compared), against the stored file elsewhere."""
import os
import sys

import numpy as np
import torch

import make_golden as MG
import refshim
import vpt_b200
from test_autograd import emulated, exact  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_autograd_golden as MAG  # noqa: E402


def _fixture():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "autograd_gradient.pt"), weights_only=False)
    if refshim.available():  # the stored file must still be what the reference computes
        live = MAG.make_autograd_gradient()
        for case in ("bc_loop", "camera"):
            assert abs(live[case]["loss"].item() - fx[case]["loss"].item()) <= 1e-5 * abs(fx[case]["loss"].item()), case
            for n, g in fx[case]["grads"].items():
                lg = live[case]["grads"][n]
                assert (g is None) == (lg is None), (case, n)
                if g is not None:
                    assert (lg["sample"] - g["sample"]).abs().max().item() <= 1e-5 * max(g["norm"].item(), 1e-12), (case, n)
        fx = live
    return fx


def _policy(fx, seed):
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), fx["policy_kwargs"], vpt_b200.PI_HEAD_KWARGS)
    pol.load_state_dict(MG.seeded_state_dict(MG.template_from(fx["schema"]), seed, fx["perturbed"]))
    return pol


def _check(pol, ref_grads, loss, ref_loss):
    """Loss to 1e-4; gradients exactly where the reference has them; norms and sampled elements to 1e-3 of the parameter's gradient norm
    outside the CNN and 5e-2 inside it (mask flips, see test_training.py)."""
    assert abs(loss - ref_loss.item()) < 1e-4 * abs(ref_loss.item())
    named = dict(pol.named_parameters())
    assert set(named) == set(ref_grads)
    n_dense = 0
    for n, ref in ref_grads.items():
        g = named[n].grad
        if ref is None:
            assert g is None, f"{n}: the reference leaves it without a gradient"
            continue
        assert g is not None and tuple(g.shape) == ref["shape"], n
        gflat = g.flatten()
        tol = 5e-2 if n.startswith("net.img_process.cnn") else 1e-3
        nrm = ref["norm"].item()
        assert abs(gflat.norm().item() - nrm) <= tol * nrm, n
        err = (gflat[MG.grad_sample_index(n, gflat.numel())] - ref["sample"]).abs().max().item()
        assert err <= tol * nrm, (n, err / nrm)
        n_dense += 1
    return n_dense


def test_reference_bc_loop_runs_unchanged(emulated, exact):
    """behavioural_cloning.py:86-123 with `set_autograd(True)`: the same calls, the same gradient."""
    fx = _fixture()
    pol = _policy(fx, fx["wseed"]).set_autograd(True)
    imgs, actions = MAG.bc_loop_inputs()
    hidden = {}
    dummy_first = torch.from_numpy(np.array((False,)))
    total = 0.0
    for i in range(MAG.SAMPLES):
        ep = MAG.EPISODES[i]
        if ep not in hidden:
            hidden[ep] = pol.initial_state(1)
        pd, _, new_state = pol.get_output_for_observation({"img": imgs[i]}, hidden[ep], dummy_first)
        log_prob = pol.get_logprob_of_action(pd, {k: v[i] for k, v in actions.items()})
        hidden[ep] = [(m if m is None else m.detach(), (k.detach(), v.detach())) for m, (k, v) in new_state]
        loss = -log_prob / MAG.SAMPLES
        total += loss.item()
        loss.backward()
    assert pol.value_head.linear.weight.grad is None
    assert _check(pol, fx["bc_loop"]["grads"], total, fx["bc_loop"]["loss"]) > 40


def test_camera_only_custom_loss(emulated, exact):
    fx = _fixture()
    pol = _policy(fx, fx["wseed"]).set_autograd(True)
    ref = _policy(fx, fx["ref_wseed"])
    img, first, actions, target = MAG.camera_inputs()
    B = img.shape[0]
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref.initial_state(B))
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    loss = MAG.camera_loss(pd, vpred, actions, pd_ref, pol.denormalize, target)
    loss.backward()
    assert pol.pi_head.buttons.linear_layer.weight.grad is None
    assert _check(pol, fx["camera"]["grads"], loss.item(), fx["camera"]["loss"]) > 40
