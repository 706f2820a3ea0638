"""RLTrainer with the entropy bonus against the reference's own autograd of the RL loss minus ent_coef * mean pi_head.entropy(pd)
(tests/golden/rl_entropy_gradient.pt, made by tools/make_rl_entropy_golden.py): the loss and its terms, sampled gradient elements and
norms of every parameter, which parameters get no gradient, and the EWMA normaliser after the call.  Live where the reference checkout is
present (the stored fixture is then also re-derived and compared), against the stored file elsewhere."""
import os
import sys

import torch

import make_golden as MG
import refshim
import vpt_b200
import vpt_oracle as O
from test_head_dist import emulated, exact  # noqa: F401  (fixtures)
from test_rl_training import NORM
from video_pre_training_b200.training import RLTrainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_rl_entropy_golden as MREG  # noqa: E402
import make_rl_golden as MRG  # noqa: E402


def _fixture():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "rl_entropy_gradient.pt"), weights_only=False)
    if refshim.available():  # the stored file must still be what the reference computes
        live = MREG.make_rl_entropy_gradient()
        assert abs(live["loss"].item() - fx["loss"].item()) <= 1e-5 * abs(fx["loss"].item())
        assert torch.allclose(live["terms"], fx["terms"], rtol=1e-5, atol=0)
        for n, g in fx["grads"].items():
            lg = live["grads"][n]
            assert (g is None) == (lg is None), n
            if g is not None:
                assert (lg["sample"] - g["sample"]).abs().max().item() <= 1e-5 * max(g["norm"].item(), 1e-12), n
        fx = live
    return fx


def test_rl_entropy_gradient_matches_reference_autograd(emulated, exact):  # noqa: F811
    """bf16 rounding off: loss to 1e-4, terms (the entropy included) to 1e-4, the normaliser to 1e-6, sampled gradient elements to 1e-3 of
    the parameter's gradient norm outside the CNN and 5e-2 inside it (as tests/test_rl_golden.py); the bonus moves the camera head's sampled
    gradient elements by three times that tolerance (checked against tests/golden/rl_gradient.pt, the same call without it)."""
    fx = _fixture()
    pkw = fx["policy_kwargs"]
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), pkw, vpt_b200.PI_HEAD_KWARGS)
    pol.load_state_dict(MG.seeded_state_dict(MG.template_from(fx["schema"]), fx["wseed"], fx["perturbed"]))
    sd_ref = MG.seeded_state_dict(MG.template_from(fx["schema"]), fx["ref_wseed"], fx["perturbed"])
    img, first, actions, _, _ = MRG.rl_inputs()
    B = img.shape[0]
    with torch.no_grad():
        (pd_ref, _, _), _ = O.agent_policy_forward(sd_ref, O.Cfg(**pkw), img, first, O.initial_state(O.Cfg(**pkw), B))
    tr = RLTrainer(pol)
    loss, _ = tr.loss_and_grad(img, first, pol.initial_state(B), actions, fx["old_logprob"], fx["advantages"], fx["returns"], pd_ref,
                               vf_coef=fx["vf_coef"], kl_coef=fx["kl_coef"], clip=fx["clip"], ent_coef=fx["ent_coef"])
    assert abs(loss.item() - fx["loss"].item()) < 1e-4 * abs(fx["loss"].item())
    terms = torch.stack([tr.stats["pi_loss"], tr.stats["vf_loss"], tr.stats["kl_ref"], tr.stats["entropy"]])
    assert torch.allclose(terms, fx["terms"], rtol=1e-4, atol=1e-6), (terms, fx["terms"])
    for k in NORM:
        assert torch.allclose(getattr(pol.value_head.normalizer, k).detach(), fx["normalizer"][k], rtol=1e-6, atol=0), k
    named = dict(pol.named_parameters())
    assert set(named) == set(fx["grads"])
    n_dense = 0
    for n, ref in fx["grads"].items():
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
    assert n_dense > 40
    plain = torch.load(os.path.join(ROOT, "tests", "golden", "rl_gradient.pt"), weights_only=False)["grads"]
    n = "pi_head.camera.linear_layer.weight"
    moved = (fx["grads"][n]["sample"] - plain[n]["sample"]).abs().max().item()
    assert moved > 3e-3 * fx["grads"][n]["norm"].item(), moved
