#!/usr/bin/env python
"""Generates tests/golden/idm_gradient.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_idm_golden.py

The reference InverseActionPolicy at the SMALL_IDM config of tests/test_idm.py (B = 2, T = 8, seeded weights with perturbed norms and
biases, seeded factored actions) with autograd: the IDM training loss -mean_{b,t} sum_sub-actions log p(action) and, per parameter,
either None (no gradient) or the gradient's shape, whether it is all zeros, its norm and a fixed element sample.  Same conventions as
oracle/make_golden.py (whose helpers it uses): no state dict is stored, the weights come back from the stored schema and seed."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402
import refshim  # noqa: E402

WSEED = 5


def idm_gradient_inputs(B=2, T=8):
    g = torch.Generator().manual_seed(6)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    actions = {"buttons": torch.randint(0, 2, (B, T, 20), generator=g), "camera": torch.randint(0, 11, (B, T, 2), generator=g)}
    return img, torch.zeros(B, T, dtype=torch.bool), actions


def make_idm_gradient():
    """The fixture as a dict (also called by tests/test_idm_golden.py for the live comparison)."""
    import vpt_b200
    from test_idm import SMALL_IDM

    ns = refshim.load()
    mapper = ns.action_mapping.IDMActionMapping(n_camera_bins=11)
    ref = ns.policy.InverseActionPolicy(action_space=ns.DictType(**mapper.get_action_space_update()), pi_head_kwargs=dict(temperature=2.0),
                                        idm_net_kwargs=vpt_b200.idm_net_kwargs(**SMALL_IDM))
    ref.load_state_dict(MG.seeded_state_dict(ref.state_dict(), WSEED, perturbed=True))
    ref.train()
    img, first, actions = idm_gradient_inputs()
    (pd, _, _), _ = ref(obs={"img": img}, first=first, state_in=ref.initial_state(img.shape[0]))
    loss = -ref.pi_head.logprob(actions, pd).mean()
    loss.backward()
    grads = {}
    for name, p in ref.named_parameters():
        if p.grad is None:
            grads[name] = None
            continue
        gflat = p.grad.detach().flatten()
        grads[name] = dict(shape=tuple(p.grad.shape), zero=bool((gflat == 0).all()), norm=gflat.norm().clone(),
                           sample=gflat[MG.grad_sample_index(name, gflat.numel())].clone() if gflat.numel() else gflat.clone())
    return dict(schema=MG.schema_of(ref.state_dict()), wseed=WSEED, perturbed=True, loss=loss.detach().clone(), grads=grads)


if __name__ == "__main__":
    MG._save("idm_gradient", make_idm_gradient())
