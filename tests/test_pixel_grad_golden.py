"""The image gradient against the reference's own autograd (tests/golden/pixel_gradient.pt, made by tools/make_pixel_golden.py):
`loss.backward()` with an `img` that requires grad, non-integer frames with values outside [0, 255], a BC loss and a camera-only loss, for
the agent with every parameter frozen, the agent with every parameter training (whose parameter gradients are compared too) and the IDM.
Live where the reference checkout is present (the stored fixture is then also re-derived and compared), against the stored file elsewhere."""
import os
import sys

import pytest
import torch

import make_golden as MG
import refshim
import vpt_b200
from test_autograd_golden import _check, _policy
from test_idm import SMALL_IDM
from test_pixel_grad import emu, emulated, exact, pix  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_pixel_golden as MPG  # noqa: E402

CASES = [f"{m}_{w}" for m in ("agent_frozen", "agent_train", "idm") for w in MPG.LOSSES]


def _fixture():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "pixel_gradient.pt"), weights_only=False)
    if refshim.available():  # the stored file must still be what the reference computes
        live = MPG.make_pixel_gradient()
        for case in CASES:
            a, b = live[case], fx[case]
            assert abs(a["loss"].item() - b["loss"].item()) <= 1e-5 * abs(b["loss"].item()), case
            assert (a["img_grad"] - b["img_grad"]).norm().item() <= 1e-5 * b["img_grad"].norm().item(), case
        fx = live
    return fx


def _check_img(g, ref):
    """The CNN's tolerance of tests/test_autograd_golden.py `_check`: norm and elements to 5e-2 of the gradient's norm (max-pool / ReLU
    mask flips), here over the whole image gradient."""
    nrm = ref.norm().item()
    assert g.shape == ref.shape and g.dtype == torch.float32
    assert abs(g.norm().item() - nrm) <= 5e-2 * nrm
    assert (g - ref).norm().item() <= 5e-2 * nrm


def _idm(fx):
    pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), vpt_b200.idm_net_kwargs(**SMALL_IDM))
    pol.load_state_dict(MG.seeded_state_dict(MG.template_from(fx["idm_schema"]), fx["wseed"], fx["perturbed"]))
    return pol


@pytest.mark.parametrize("which", MPG.LOSSES)
@pytest.mark.parametrize("model", ["agent_frozen", "agent_train", "idm"])
def test_image_gradient_matches_reference_autograd(pix, exact, model, which):  # noqa: F811
    fx = _fixture()
    ref = fx[f"{model}_{which}"]
    if model == "idm":
        pol, (img, first, actions) = _idm(fx), MPG.idm_inputs()
    else:
        pol, (img, first, actions) = _policy(fx, fx["wseed"]), MPG.agent_inputs()
    pol.set_autograd(True)
    if model != "agent_train":
        pol.requires_grad_(False)
    x = img.clone().requires_grad_(True)
    (pd, _, _), _ = pol({"img": x}, first, pol.initial_state(img.shape[0]))
    loss = MPG.loss_of(pd, actions, which)
    loss.backward()
    _check_img(x.grad, ref["img_grad"])
    if model == "agent_train":
        assert _check(pol, ref["grads"], loss.item(), ref["loss"]) > 40
    else:
        assert abs(loss.item() - ref["loss"].item()) < 1e-4 * abs(ref["loss"].item())
        assert all(p.grad is None for p in pol.parameters())
