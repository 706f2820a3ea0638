#!/usr/bin/env python
"""Generates tests/golden/pixel_gradient.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_pixel_golden.py

The reference's own autograd of d loss / d img: its ImgPreprocessing (lib/policy.py:39-45) is img.to(float32) / 255, so a float leaf
gets the gradient through the whole model.  Non-integer frames with values outside [0, 255], at the SMALL configs of tests/common.py
(agent, B = 2, T = 4) and tests/test_idm.py (IDM, B = 1, T = 8), seeded weights with perturbed norms and biases:

    agent_frozen   every parameter frozen (requires_grad_(False))
    agent_train    every parameter training (their gradients are stored too)
    idm            the IDM, every parameter frozen

each with two losses: `bc` (-mean over frames of the summed log-probabilities of the taken actions, every sub-action for the IDM) and
`camera` (the same for the camera head alone).  Per case: the loss and the full image gradient (fp32 [B, T, H, W, 3]), and for
agent_train per parameter the gradient's norm and a fixed element sample.  No state dict is stored."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402
import refshim  # noqa: E402
from make_autograd_golden import _grads  # noqa: E402

WSEED = 7
LOSSES = ("bc", "camera")


def agent_inputs():
    g = torch.Generator().manual_seed(41)
    B, T = 2, 4
    img = torch.rand((B, T, 32, 32, 3), generator=g) * 340.0 - 40.0  # non-integer, some below 0 and above 255
    first = torch.zeros(B, T, dtype=torch.bool)
    first[1, 2] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    return img, first, actions


def idm_inputs():
    g = torch.Generator().manual_seed(42)
    B, T = 1, 8
    img = torch.rand((B, T, 32, 32, 3), generator=g) * 340.0 - 40.0
    actions = {"buttons": torch.randint(0, 2, (B, T, 20), generator=g), "camera": torch.randint(0, 11, (B, T, 2), generator=g)}
    return img, torch.zeros(B, T, dtype=torch.bool), actions


def loss_of(pd, actions, which):
    """-mean over the frames of the summed log-probabilities of the taken (sub-)actions, as a plain gather over the last axis of pd, so
    that the reference's pd and this project's give the same loss whatever their leading shapes.  which: "bc" (every head) or "camera"."""
    n = actions["camera"].shape[0] * actions["camera"].shape[1]
    heads = ("camera", "buttons") if which == "bc" else ("camera",)
    return -sum(pd[k].reshape(-1, pd[k].shape[-1]).gather(-1, actions[k].reshape(-1, 1)).sum() for k in heads) / n


def _ref_idm():
    import vpt_b200
    from test_idm import SMALL_IDM

    ns = refshim.load()
    mapper = ns.action_mapping.IDMActionMapping(n_camera_bins=11)
    ref = ns.policy.InverseActionPolicy(action_space=ns.DictType(**mapper.get_action_space_update()), pi_head_kwargs=dict(temperature=2.0),
                                        idm_net_kwargs=vpt_b200.idm_net_kwargs(**SMALL_IDM))
    ref.load_state_dict(MG.seeded_state_dict(ref.state_dict(), WSEED, perturbed=True))
    return ref


def _case(pol, img, first, actions, which, train):
    for p in pol.parameters():
        p.requires_grad_(train)
        p.grad = None
    x = img.clone().requires_grad_(True)
    (pd, _, _), _ = pol({"img": x}, first, pol.initial_state(img.shape[0]))
    loss = loss_of(pd, actions, which)
    loss.backward()
    out = dict(loss=loss.detach().clone(), img_grad=x.grad.detach().clone())
    if train:
        out["grads"] = _grads(pol)
    return out


def make_pixel_gradient():
    """The fixture as a dict (also called by tests/test_pixel_grad_golden.py for the live comparison)."""
    from common import small_kwargs

    pkw = small_kwargs()
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    out = dict(policy_kwargs=pkw, wseed=WSEED, perturbed=True, schema=MG.schema_of(pol.state_dict()))
    img, first, actions = agent_inputs()
    for which in LOSSES:
        out[f"agent_frozen_{which}"] = _case(pol, img, first, actions, which, train=False)
        out[f"agent_train_{which}"] = _case(MG._ref_policy(pkw, WSEED, perturbed=True), img, first, actions, which, train=True)
    ref = _ref_idm()
    ref.train()
    out["idm_schema"] = MG.schema_of(ref.state_dict())
    img, first, actions = idm_inputs()
    for which in LOSSES:
        out[f"idm_{which}"] = _case(ref, img, first, actions, which, train=False)
    return out


if __name__ == "__main__":
    MG._save("pixel_gradient", make_pixel_gradient())
