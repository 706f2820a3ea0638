#!/usr/bin/env python
"""Generates tests/golden/autograd_gradient.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_autograd_golden.py

Two cases at the SMALL config of tests/common.py (seeded weights with perturbed norms and biases), each with the reference's own autograd:

    bc_loop   the inner loop of behavioural_cloning.py:86-123 as written: SAMPLES samples of one frame each (B = 1, T = 1) from two
              interleaved episodes, each episode's state carried and detached, `(-log_prob / BATCH_SIZE).backward()` per sample
    camera    a loss on the camera head only, over a B = 2, T = 8 batch with an episode start mid-batch: the NLL minus an entropy bonus
              plus KL_COEF * KL(pd_ref || pd) (a differently seeded frozen policy) plus an MSE on value_head.denormalize(vpred)

Per case it stores the loss, per parameter the gradient's norm and a fixed element sample (or None).  No state dict is stored."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402

WSEED, REF_WSEED = 5, 11
SAMPLES = 6           # behavioural_cloning.py's BATCH_SIZE for this fixture
EPISODES = (0, 1, 0, 1, 1, 0)
KL_COEF, ENT_COEF = 0.3, 0.05


def bc_loop_inputs():
    g = torch.Generator().manual_seed(21)
    imgs = torch.randint(0, 256, (SAMPLES, 1, 32, 32, 3), dtype=torch.uint8, generator=g)
    actions = {"camera": torch.randint(0, 121, (SAMPLES, 1, 1), generator=g), "buttons": torch.randint(0, 8641, (SAMPLES, 1, 1), generator=g)}
    return imgs, actions


def camera_inputs(B=2, T=8):
    g = torch.Generator().manual_seed(22)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    first[0, 2] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    target = 2.0 * torch.randn(B, T, generator=g)
    return img, first, actions, target


def camera_loss(pd, vpred, actions, pd_ref, denorm, target):
    """The NLL minus an entropy bonus plus a KL on the camera head, and an MSE on the denormalised value."""
    lp = pd["camera"]
    nll = -lp.gather(-1, actions["camera"].unsqueeze(-1)).squeeze(-1).sum(-1).mean()
    ent = -(torch.exp(lp) * lp).sum(-1).mean()
    kl = (torch.exp(pd_ref["camera"]) * (pd_ref["camera"] - lp)).sum(-1).mean()
    mse = ((denorm(vpred)[..., 0] - target) ** 2).mean()
    return nll - ENT_COEF * ent + KL_COEF * kl + mse


def _grads(pol):
    out = {}
    for name, p in pol.named_parameters():
        if p.grad is None:
            out[name] = None
            continue
        gflat = p.grad.detach().flatten()
        out[name] = dict(shape=tuple(p.grad.shape), norm=gflat.norm().clone(), sample=gflat[MG.grad_sample_index(name, gflat.numel())].clone())
    return out


def make_autograd_gradient():
    """The fixture as a dict (also called by tests/test_autograd_golden.py for the live comparison)."""
    from common import small_kwargs

    pkw = small_kwargs()
    # -- behavioural_cloning.py:86-123 with B = 1, T = 1 per call
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    imgs, actions = bc_loop_inputs()
    hidden = {}
    dummy_first = torch.from_numpy(__import__("numpy").array((False,)))
    total = 0.0
    for i in range(SAMPLES):
        ep = EPISODES[i]
        if ep not in hidden:
            hidden[ep] = pol.initial_state(1)
        obs = {"img": imgs[i]}
        pd, _, new_state = pol.get_output_for_observation(obs, hidden[ep], dummy_first)
        log_prob = pol.get_logprob_of_action(pd, {k: v[i] for k, v in actions.items()})
        hidden[ep] = [(m if m is None else m.detach(), (k.detach(), v.detach())) for m, (k, v) in new_state]
        loss = -log_prob / SAMPLES
        total += loss.item()
        loss.backward()
    bc = dict(loss=torch.tensor(total), grads=_grads(pol))
    # -- the camera-only custom loss
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    ref = MG._ref_policy(pkw, REF_WSEED, perturbed=True)
    img, first, cam_actions, target = camera_inputs()
    B = img.shape[0]
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref.initial_state(B))
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    loss = camera_loss(pd, vpred, cam_actions, pd_ref, pol.value_head.denormalize, target)
    loss.backward()
    cam = dict(loss=loss.detach().clone(), grads=_grads(pol))
    return dict(policy_kwargs=pkw, schema=MG.schema_of(pol.state_dict()), wseed=WSEED, ref_wseed=REF_WSEED, perturbed=True, bc_loop=bc, camera=cam)


if __name__ == "__main__":
    MG._save("autograd_gradient", make_autograd_gradient())
