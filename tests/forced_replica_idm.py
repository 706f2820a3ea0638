"""TEST INFRASTRUCTURE: the forced replica of tests/forced_replica.py for the IDM step (IDMTrainer): every layer recomputed in fp32 by
torch from the parameters, its value replaced by the taped CUDA activation (straight-through) and every ReLU / max-pool mask taken
from the tape, so that autograd returns the exact gradient at the CUDA forward's operating point.

Differences from the policy replica: the conv3d pre-stage (its output is taped as stack 0's `x_in`), stack 0's normalised first conv,
unmasked attention without KV memory or relative term, no lastlayer (lib/policy.py:389-392), factored heads."""
import torch
import torch.nn.functional as F

import vpt_oracle as O
from forced_replica import _nchw, _relu_forced, _sub


def forced_loss_idm(sd, cfg, tape, img_u8, actions, temperature=2.0, pfx="net"):
    B, t = img_u8.shape[:2]
    N = B * t
    h = cfg.hidsize
    x3 = O.conv3d_stage(O.img_preprocess(img_u8), sd, "net.conv3d_layer")             # (B, T, H, W, C), post-ReLU
    x = x3.reshape(N, *x3.shape[2:]).permute(0, 3, 1, 2)
    p = f"{pfx}.img_process.cnn"
    for i, rec in enumerate(tape["stacks"]):
        s = f"{p}.stacks.{i}"
        x = _relu_forced(x, _nchw(rec["x_in"])) if i == 0 else x
        u = F.group_norm(x, 1, sd[f"{s}.firstconv.norm.weight"], sd[f"{s}.firstconv.norm.bias"], eps=1e-5)
        full = _relu_forced(F.conv2d(u, sd[f"{s}.firstconv.layer.weight"], None, padding=1), _nchw(rec["full"]))
        y1 = _sub(F.max_pool2d(full, 3, 2, 1), _nchw(rec["y1"]))
        x = _sub(F.group_norm(y1, 1, sd[f"{s}.n.weight"], sd[f"{s}.n.bias"], eps=1e-5), _nchw(rec["x0"]))
        for j, blk in enumerate(rec["blocks"]):
            q = f"{s}.blocks.{j}"
            u = F.group_norm(x, 1, sd[f"{q}.conv0.norm.weight"], sd[f"{q}.conv0.norm.bias"], eps=1e-5)
            hmid = _relu_forced(F.conv2d(u, sd[f"{q}.conv0.layer.weight"], None, padding=1), _nchw(blk["h"]))
            u = F.group_norm(hmid, 1, sd[f"{q}.conv1.norm.weight"], sd[f"{q}.conv1.norm.bias"], eps=1e-5)
            r = _relu_forced(F.conv2d(u, sd[f"{q}.conv1.layer.weight"], None, padding=1), _nchw(blk["r"]))
            x = _sub(x + r, _nchw(blk["x"]))
    x = x.reshape(N, -1)
    u = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.dense.norm.weight"], sd[f"{p}.dense.norm.bias"], eps=1e-5)
    xd = _relu_forced(F.linear(u, sd[f"{p}.dense.layer.weight"]), tape["xd"].float())
    q = f"{pfx}.img_process.linear"
    u = F.layer_norm(xd, (xd.shape[-1],), sd[f"{q}.norm.weight"], sd[f"{q}.norm.bias"], eps=1e-5)
    x = _relu_forced(F.linear(u, sd[f"{q}.layer.weight"]), tape["x0"].float())
    heads = cfg.heads
    nl = len(tape["blocks"])
    for l, S in enumerate(tape["blocks"]):
        b = f"{pfx}.recurrent_layer.blocks.{l}"
        o = f"{b}.r.orc_block"
        xhat = _sub(F.layer_norm(x, (h,), sd[f"{b}.pre_r_ln.weight"], sd[f"{b}.pre_r_ln.bias"], eps=1e-5), S["xhat"].float())
        qv = _sub(F.linear(xhat, sd[f"{o}.q_layer.weight"], sd[f"{o}.q_layer.bias"]), S["q"].float())
        k = _sub(F.linear(xhat, sd[f"{o}.k_layer.weight"]).reshape(B, t, h), S["full_k"].float())
        v = _sub(F.linear(xhat, sd[f"{o}.v_layer.weight"]).reshape(B, t, h), S["full_v"].float())
        # R = r_layer(x_hat) meets the empty band of b_nd (10, 0): a zero bias that still carries (zero) gradient to r_layer / b_nd
        R = F.linear(xhat, sd[f"{o}.r_layer.weight"], sd[f"{o}.r_layer.bias"])
        Q, K, V = O.split_heads(qv.reshape(B, t, h), heads), O.split_heads(k, heads), O.split_heads(v, heads)
        rel = torch.einsum("btn,nd->btd", O.split_heads(R.reshape(B, t, -1), heads), sd[f"{o}.b_nd"]).sum(-1, keepdim=True)
        e = Q.shape[2]
        Wt = torch.softmax(torch.baddbmm(rel.expand(-1, -1, t), Q, K.transpose(-1, -2), alpha=1.0 / e), dim=2)
        A = torch.einsum("btp,bpe->bte", Wt, V).reshape(B, heads, t, e).permute(0, 2, 1, 3).reshape(N, h)
        A = _sub(A, S["a"].float())
        y = _sub(xhat + F.linear(A, sd[f"{o}.proj_layer.weight"], sd[f"{o}.proj_layer.bias"]), S["y"].float())
        u = F.layer_norm(y, (h,), sd[f"{b}.mlp0.norm.weight"], sd[f"{b}.mlp0.norm.bias"], eps=1e-5)
        hm = _relu_forced(F.linear(u, sd[f"{b}.mlp0.layer.weight"]), S["hmid"].float())
        z = y + F.linear(hm, sd[f"{b}.mlp1.layer.weight"], sd[f"{b}.mlp1.layer.bias"])
        x = _relu_forced(z, S["z"].float()) if l == nl - 1 else _sub(z, S["z"].float())
    lat = F.layer_norm(x, (h,), sd[f"{pfx}.final_ln.weight"], sd[f"{pfx}.final_ln.bias"], eps=1e-5)
    lat = _sub(lat, lat.detach().to(torch.bfloat16))  # the heads read the bf16 latent
    logp = 0.0
    for name, n in (("buttons", 2), ("camera", 11)):
        lin = f"pi_head.{name}.linear_layer"
        lg = F.linear(lat, sd[f"{lin}.weight"], sd[f"{lin}.bias"]).float().reshape(N, -1, n) / temperature
        lg = F.log_softmax(lg, dim=-1)
        logp = logp + lg.gather(-1, actions[name].reshape(N, -1, 1).to(torch.int64)).squeeze(-1).sum(-1)
    return -logp.mean()
