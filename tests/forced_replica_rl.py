"""TEST INFRASTRUCTURE: the RL loss (tests/test_rl_training.py, rl_loss) through the forced replica of tests/forced_replica.py, i.e. autograd
at the CUDA forward's operating point.  The replica's latent is taken where its BC loss reads it (the first head's linear layer), so the
network part stays the one `forced_loss` defines; the heads, the value head and the RL loss are then computed from it here."""
import types

import torch
import torch.nn.functional as F

import forced_replica
from test_rl_training import rl_loss


def forced_latent(sd, cfg, tape, img_u8, first, actions, temperature=2.0):
    """The latent (bf16-valued, fp32 gradient) of `forced_replica.forced_loss` with the same arguments."""
    seen = {}

    def linear(x, w, b=None):
        if w is sd["pi_head.camera.linear_layer.weight"]:
            seen["lat"] = x
        return F.linear(x, w, b)

    shim = types.SimpleNamespace(**{k: getattr(F, k) for k in dir(F) if not k.startswith("_")})
    shim.linear = linear
    saved = forced_replica.F
    forced_replica.F = shim
    try:
        forced_replica.forced_loss(sd, cfg, tape, img_u8, first, actions, temperature)
    finally:
        forced_replica.F = saved
    return seen["lat"]


def forced_rl_loss(sd, cfg, tape, img_u8, first, actions, old_lp, adv, returns, pd_ref, norm, vf_coef, kl_coef, clip, temperature=2.0):
    """The RL loss at the taped operating point; `norm` (the normaliser's three values before the call) is updated in place."""
    lat = forced_latent(sd, cfg, tape, img_u8, first, actions, temperature)
    B, t = img_u8.shape[:2]
    pd = {}
    for name in ("camera", "buttons"):
        lin = f"pi_head.{name}.linear_layer"
        lg = F.log_softmax(F.linear(lat, sd[f"{lin}.weight"], sd[f"{lin}.bias"]).float() / temperature, dim=-1)
        pd[name] = lg.reshape(B, t, 1, -1)
    vpred = F.linear(lat, sd["value_head.linear.weight"], sd["value_head.linear.bias"]).reshape(B, t, 1)
    return rl_loss(pd, vpred, actions, old_lp, adv, returns, pd_ref, norm, vf_coef, kl_coef, clip)
