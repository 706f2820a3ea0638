#!/usr/bin/env python
"""Generates tests/golden/rl_entropy_gradient.pt from the UNMODIFIED reference (run where its checkout exists, see oracle/refshim.py):

    python tools/make_rl_entropy_golden.py

The RL loss of tools/make_rl_golden.py (same policies, inputs and coefficients) with the entropy bonus from the reference's own pi_head:

    loss  = L_pi + vf_coef * L_v + kl_coef * L_kl - ent_coef * mean pi_head.entropy(pd)

It stores what make_rl_golden.py stores, the entropy term among the loss's terms, and ent_coef.  No state dict is stored."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import make_golden as MG  # noqa: E402
import make_rl_golden as MRG  # noqa: E402

ENT_COEF = 2.0  # large enough that the bonus moves the camera head's gradient to several times the test's tolerance


def make_rl_entropy_gradient():
    """The fixture as a dict (also called by tests/test_rl_entropy_golden.py for the live comparison)."""
    from common import small_kwargs

    pkw = small_kwargs()
    pol = MG._ref_policy(pkw, MRG.WSEED, perturbed=True)
    ref = MG._ref_policy(pkw, MRG.REF_WSEED, perturbed=True)
    pol.train()
    img, first, actions, adv, returns = MRG.rl_inputs()
    B, T = img.shape[:2]
    N = B * T
    flat = lambda pd: {k: v.reshape(N, 1, *v.shape[2:]) for k, v in pd.items()}
    fa = {k: v.reshape(N, 1) for k, v in actions.items()}
    with torch.no_grad():
        (pd_ref, _, _), _ = ref({"img": img}, first, ref.initial_state(B))
        (pd0, _, _), _ = pol({"img": img}, first, pol.initial_state(B))
        old = pol.get_logprob_of_action(flat(pd0), fa).reshape(B, T) - torch.log(torch.tensor(MRG.RATIOS).repeat(N // len(MRG.RATIOS)).reshape(B, T))
    (pd, vpred, _), _ = pol({"img": img}, first, pol.initial_state(B))
    ratio = torch.exp(pol.get_logprob_of_action(flat(pd), fa).reshape(B, T) - old)
    l_pi = -torch.min(ratio * adv, ratio.clamp(1 - MRG.CLIP, 1 + MRG.CLIP) * adv).mean()
    l_v = pol.value_head.loss(vpred, returns[..., None])
    l_kl = pol.get_kl_of_action_dists(pd_ref, pd).mean()
    ent = pol.pi_head.entropy(pd).mean()
    loss = l_pi + MRG.VF_COEF * l_v + MRG.KL_COEF * l_kl - ENT_COEF * ent
    loss.backward()
    grads = {}
    for name, p in pol.named_parameters():
        if p.grad is None:
            grads[name] = None
            continue
        gflat = p.grad.detach().flatten()
        grads[name] = dict(shape=tuple(p.grad.shape), norm=gflat.norm().clone(), sample=gflat[MG.grad_sample_index(name, gflat.numel())].clone())
    nz = pol.value_head.normalizer
    return dict(policy_kwargs=pkw, schema=MG.schema_of(pol.state_dict()), wseed=MRG.WSEED, ref_wseed=MRG.REF_WSEED, perturbed=True,
                vf_coef=MRG.VF_COEF, kl_coef=MRG.KL_COEF, ent_coef=ENT_COEF, clip=MRG.CLIP, old_logprob=old.detach().clone(),
                advantages=adv.clone(), returns=returns.clone(), loss=loss.detach().clone(),
                terms=torch.stack([l_pi, l_v, l_kl, ent]).detach().clone(), grads=grads,
                normalizer={k: getattr(nz, k).detach().clone() for k in ("running_mean", "running_mean_sq", "debiasing_term")})


if __name__ == "__main__":
    MG._save("rl_entropy_gradient", make_rl_entropy_gradient())
