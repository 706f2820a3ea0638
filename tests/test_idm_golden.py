"""IDMTrainer against the reference's own autograd (tests/golden/idm_gradient.pt, made by tools/make_idm_golden.py): the loss, sampled
gradient elements and norms of every parameter, and which parameters get no gradient (None), exact zeros or an empty gradient.  Live
where the reference checkout is present (the stored fixture is then also re-derived and compared), against the stored file elsewhere."""
import os
import sys

import torch

import make_golden as MG
import refshim
import vpt_b200
from test_idm import SMALL_IDM
from test_idm_training import emulated, exact  # noqa: F401  (fixtures)
from video_pre_training_b200.training import IDMTrainer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_idm_golden as MIG  # noqa: E402


def _fixture():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "idm_gradient.pt"), weights_only=False)
    if refshim.available():  # the stored file must still be what the reference computes
        live = MIG.make_idm_gradient()
        assert abs(live["loss"].item() - fx["loss"].item()) <= 1e-5 * abs(fx["loss"].item())
        for n, g in fx["grads"].items():
            lg = live["grads"][n]
            assert (g is None) == (lg is None), n
            if g is not None:
                assert lg["shape"] == g["shape"] and lg["zero"] == g["zero"], n
                assert g["sample"].numel() == 0 or (lg["sample"] - g["sample"]).abs().max().item() <= 1e-5 * max(g["norm"].item(), 1e-12), n
        fx = live
    return fx


def test_idm_gradient_matches_reference_autograd(emulated, exact):
    """bf16 rounding off (the function the reference computes): loss to 1e-4; the None / zero / empty pattern exactly; sampled
    elements to 1e-3 of the parameter's gradient norm outside the CNN, 5e-2 inside it (mask flips, see test_idm_training.py)."""
    fx = _fixture()
    kw = vpt_b200.idm_net_kwargs(**SMALL_IDM)
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), kw)
    pol.load_state_dict(MG.seeded_state_dict(MG.template_from(fx["schema"]), fx["wseed"], fx["perturbed"]))
    img, first, actions = MIG.idm_gradient_inputs()
    loss, _ = IDMTrainer(pol).loss_and_grad(img, first, pol.initial_state(img.shape[0]), actions)
    assert abs(loss.item() - fx["loss"].item()) < 1e-4 * abs(fx["loss"].item())
    named = dict(pol.named_parameters())
    assert set(named) == set(fx["grads"])
    n_dense = 0
    for n, ref in fx["grads"].items():
        g = named[n].grad
        if ref is None:
            assert g is None, f"{n}: the reference leaves it without a gradient"
            continue
        assert g is not None and tuple(g.shape) == ref["shape"], n
        if ref["zero"]:
            assert not g.any(), f"{n}: the reference's gradient is all zeros"
            continue
        gflat = g.flatten()
        tol = 5e-2 if n.startswith(("net.img_process.cnn.stacks", "net.conv3d_layer")) else 1e-3
        nrm = ref["norm"].item()
        assert abs(gflat.norm().item() - nrm) <= tol * nrm, n
        err = (gflat[MG.grad_sample_index(n, gflat.numel())] - ref["sample"]).abs().max().item()
        assert err <= tol * nrm, (n, err / nrm)
        n_dense += 1
    assert n_dense > 80
