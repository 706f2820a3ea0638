#!/usr/bin/env python
"""Generates tests/golden/rl_gradient.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_rl_golden.py

The reference MinecraftAgentPolicy at the SMALL config of tests/common.py (B = 2, T = 8 with an episode start mid-batch, seeded
weights with perturbed norms and biases) and a differently seeded, perturbed copy as the frozen reference policy, with autograd of the
RL loss composed from the reference's own methods:

    lp    = get_logprob_of_action(pd, a)                 (frames as the batch: the method handles one step per row)
    loss  = -mean min(ratio A, clamp(ratio, 0.8, 1.2) A) + vf_coef * value_head.loss(vpred, returns)   (train mode: updates the normaliser)
            + kl_coef * mean get_kl_of_action_dists(pd_ref, pd)

It stores the inputs that are not seeded here (old_logprob, advantages, returns), the loss, per parameter the gradient's norm and a
fixed element sample (or None), and the normaliser's three values after the call.  No state dict is stored (oracle/make_golden.py)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402

WSEED, REF_WSEED = 3, 9
VF_COEF, KL_COEF, CLIP = 0.5, 0.1, 0.2
RATIOS = (0.5, 0.7, 0.9, 1.0, 1.1, 1.35, 1.6, 0.75)  # per row: clipped on both sides and not, none on a boundary
ADV_SIGNS = (1.0, -1.0, 1.0, -1.0, -1.0, 1.0, -1.0, -1.0)


def rl_inputs(B=2, T=8):
    g = torch.Generator().manual_seed(12)
    img = torch.randint(0, 256, (B, T, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(B, T, dtype=torch.bool)
    first[1, 3] = True
    actions = {"camera": torch.randint(0, 121, (B, T, 1), generator=g), "buttons": torch.randint(0, 8641, (B, T, 1), generator=g)}
    adv = torch.tensor(ADV_SIGNS).repeat(B * T // len(ADV_SIGNS)).reshape(B, T) * (0.5 + torch.rand(B, T, generator=g))
    returns = 3.0 + 2.0 * torch.randn(B, T, generator=g)
    return img, first, actions, adv, returns


def make_rl_gradient():
    """The fixture as a dict (also called by tests/test_rl_golden.py for the live comparison)."""
    from common import small_kwargs

    pkw = small_kwargs()
    pol = MG._ref_policy(pkw, WSEED, perturbed=True)
    ref = MG._ref_policy(pkw, REF_WSEED, perturbed=True)
    pol.train()
    img, first, actions, adv, returns = rl_inputs()
    B, T = img.shape[:2]
    N = B * T
    flat = lambda pd: {k: v.reshape(N, 1, *v.shape[2:]) for k, v in pd.items()}
    fa = {k: v.reshape(N, 1) for k, v in actions.items()}
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref.initial_state(B))
        (pd0, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
        old = pol.get_logprob_of_action(flat(pd0), fa).reshape(B, T) - torch.log(torch.tensor(RATIOS).repeat(N // len(RATIOS)).reshape(B, T))
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    ratio = torch.exp(pol.get_logprob_of_action(flat(pd), fa).reshape(B, T) - old)
    l_pi = -torch.min(ratio * adv, ratio.clamp(1 - CLIP, 1 + CLIP) * adv).mean()
    l_v = pol.value_head.loss(vpred, returns[..., None])
    l_kl = pol.get_kl_of_action_dists(pd_ref, pd).mean()
    loss = l_pi + VF_COEF * l_v + KL_COEF * l_kl
    loss.backward()
    grads = {}
    for name, p in pol.named_parameters():
        if p.grad is None:
            grads[name] = None
            continue
        gflat = p.grad.detach().flatten()
        grads[name] = dict(shape=tuple(p.grad.shape), norm=gflat.norm().clone(), sample=gflat[MG.grad_sample_index(name, gflat.numel())].clone())
    nz = pol.value_head.normalizer
    return dict(policy_kwargs=pkw, schema=MG.schema_of(pol.state_dict()), wseed=WSEED, ref_wseed=REF_WSEED, perturbed=True,
                vf_coef=VF_COEF, kl_coef=KL_COEF, clip=CLIP, old_logprob=old.detach().clone(), advantages=adv.clone(), returns=returns.clone(),
                loss=loss.detach().clone(), terms=torch.stack([l_pi, l_v, l_kl]).detach().clone(), grads=grads,
                normalizer={k: getattr(nz, k).detach().clone() for k in ("running_mean", "running_mean_sq", "debiasing_term")})


if __name__ == "__main__":
    MG._save("rl_gradient", make_rl_gradient())
