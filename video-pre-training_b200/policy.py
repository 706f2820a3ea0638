"""Drop-in replacements for the reference's policy classes (lib/policy.py) whose forward pass runs entirely in the
hand-written sm_90a kernels of libvpt_b200.so.

    MinecraftPolicy        lib/policy.py:83-224    forward(ob, state_in, context) / initial_state / output_latent_size
    MinecraftAgentPolicy   lib/policy.py:227-339   forward / act / get_output_for_observation / get_logprob_of_action /
                                                   get_kl_of_action_dists / v / initial_state
    InverseActionPolicy    lib/policy.py:406-467   (see idm.py)
    pi_head                lib/action_head.py:136-260  logprob / sample / entropy / kl_divergence, on the dict and on each sub-head

Same constructor kwargs, same state pytree (list over layers of (state_mask bool (B,1,maxlen) | None, (K, V) fp32
(B,maxlen,hidsize))), same `state_dict()` keys / shapes (SURVEY.md App. B), so reference weight files load with
`load_state_dict`.  Parameters are kept in fp32 exactly as the reference stores them; at first use (and whenever a
parameter changes) they are re-laid-out for the kernels (`_Prepared`): conv weights OIHW -> [Cout][tap][Cin] bf16 with
the input GroupNorm gamma folded in plus the 9 border-class fold tables, linear weights with LayerNorm folded, the
`dense` columns permuted from C,H,W to H,W,C order.

`encode(img)` runs the CNN part (frames -> the `dense` layer's output and its row statistics, `FrameLatents`) on its own, and
`forward({"img_latent": latents}, ...)` the rest of the network from them.

`forward` runs under no_grad and returns detached tensors; the trainers have their own hand-written backward (training.py).
After `set_autograd(True)` a forward in grad mode (with a parameter that requires grad) is instead an autograd `Function` on that
same backward, so that `loss.backward()` trains the model (training._AutogradRunner).  There is no CPU path: CPU tensors raise.
"""
import functools
import math
import weakref
from collections import OrderedDict
from typing import Dict, Optional

import torch
from torch import nn

from . import _native as nat
from . import ops
from .types import DictType

BF16, F32 = torch.bfloat16, torch.float32
NBASIS = 10  # lib/xf.py:259


# ---------------------------------------------------------------------------------------------------------------
# parameter schema + init (names / shapes / init scales of the reference)
# ---------------------------------------------------------------------------------------------------------------
class _Node(nn.Module):
    """Bare container so that `state_dict()` keys nest exactly like the reference's module tree."""


def _set(root: nn.Module, name: str, tensor: torch.Tensor, requires_grad=True):
    parts = name.split(".")
    m = root
    for p in parts[:-1]:
        if p not in m._modules:
            m.add_module(p, _Node())
        m = m._modules[p]
    m.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=requires_grad))


def _fanin(shape, scale):
    """lib/util.py:67-73 / lib/torch_util.py:79: default torch init, then every output row L2-normalised to `scale`."""
    w = torch.empty(shape)
    nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    flat = w.reshape(shape[0], -1)
    flat *= scale / flat.norm(dim=1, p=2, keepdim=True)
    return w


def _default_linear(out_f, in_f):
    """nn.Linear default init (lib/action_head.py:150, lib/scaled_mse_head.py:24)."""
    w = torch.empty(out_f, in_f)
    nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    bound = 1 / math.sqrt(in_f)
    return w, torch.empty(out_f).uniform_(-bound, bound)


class NetConfig:
    """The kwargs of lib/policy.py:96-126 that the transformer models use (agent.py:16-36)."""

    def __init__(self, recurrence_type="transformer", impala_width=1, impala_chans=(16, 32, 32), obs_processing_width=256,
                 hidsize=512, single_output=False, img_shape=None, scale_input_img=True, only_img_input=False,
                 init_norm_kwargs=None, impala_kwargs=None, input_shape=None, active_reward_monitors=None, img_statistics=None,
                 first_conv_norm=False, diff_mlp_embedding=False, attention_mask_style="clipped_causal", attention_heads=8,
                 attention_memory_size=2048, use_pointwise_layer=True, pointwise_ratio=4, pointwise_use_activation=False,
                 n_recurrence_layers=1, recurrence_is_residual=True, timesteps=None, use_pre_lstm_ln=True, conv3d_params=None,
                 **unused_kwargs):
        init_norm_kwargs = init_norm_kwargs or {}
        impala_kwargs = impala_kwargs or {}
        # Only the configuration family of the released models is implemented in CUDA; anything else is refused loudly.
        if recurrence_type != "transformer":
            raise NotImplementedError("vpt_b200: only recurrence_type='transformer' (all released VPT models, agent.py:32)")
        if init_norm_kwargs.get("group_norm_groups", None) != 1 or init_norm_kwargs.get("batch_norm", False):
            raise NotImplementedError("vpt_b200: init_norm_kwargs must be {'batch_norm': False, 'group_norm_groups': 1} (agent.py:26)")
        if impala_kwargs.get("post_pool_groups", None) != 1:
            raise NotImplementedError("vpt_b200: impala_kwargs must be {'post_pool_groups': 1} (agent.py:24)")
        if img_statistics is not None or not scale_input_img or diff_mlp_embedding or use_pre_lstm_ln:
            raise NotImplementedError("vpt_b200: img_statistics / scale_input_img=False / diff_mlp_embedding / use_pre_lstm_ln unsupported")
        if not (use_pointwise_layer and recurrence_is_residual) or pointwise_use_activation:
            raise NotImplementedError("vpt_b200: needs use_pointwise_layer, recurrence_is_residual, no pointwise activation")
        if attention_mask_style not in ("clipped_causal", "none"):
            raise AssertionError("mask must be 'none' or 'clipped_causal'")  # lib/masked_attention.py:134
        assert attention_memory_size >= 0  # lib/masked_attention.py:135
        self.chans = tuple(int(impala_width * c) for c in impala_chans)
        self.hidsize = hidsize
        self.heads = attention_heads
        self.timesteps = timesteps
        self.maxlen = attention_memory_size - timesteps
        self.mask_style = attention_mask_style
        self.n_layers = n_recurrence_layers
        self.img_shape = tuple(img_shape)
        self.pointwise_ratio = pointwise_ratio
        self.single_output = single_output
        # IDM (lib/policy.py:342-372): a temporal conv3d pre-stage feeds the CNN, whose first conv is then normalised too
        self.conv3d_out = None
        if conv3d_params is not None:
            ks, pad = list(conv3d_params.get("kernel_size", [])), list(conv3d_params.get("padding", []))
            if conv3d_params.get("inchan") != 3 or ks != [5, 1, 1] or pad != [2, 0, 0]:
                raise NotImplementedError("vpt_b200: conv3d_params must be inchan=3, kernel_size=[5,1,1], padding=[2,0,0] (the IDM)")
            self.conv3d_out = int(conv3d_params["outchan"])
            first_conv_norm = True
        self.first_conv_norm = first_conv_norm
        self.cnn_outsize = 256
        assert hidsize % attention_heads == 0, "Embsize must be divisible by number of heads"  # lib/xf.py:98
        if hidsize // attention_heads != 128:
            raise NotImplementedError("vpt_b200: head_dim must be 128 (true of every VPT width)")
        assert self.maxlen > 0 or self.mask_style == "none"  # lib/xf.py:256
        H, W, Cin = self.img_shape
        want_cin = 3 if self.conv3d_out is None else self.conv3d_out
        if Cin != want_cin or H % 16 or W % 16 or any(c % 64 for c in self.chans) or (self.conv3d_out or 64) % 64:
            raise NotImplementedError("vpt_b200: img must be (H,W,3) [(H,W,conv3d outchan) for the IDM] with H,W % 16 == 0 and channels % 64 == 0")
        if self.first_conv_norm and self.conv3d_out is None:
            raise NotImplementedError("vpt_b200: first_conv_norm without the conv3d pre-stage is not implemented")
        self.final_hw = (H // 8, W // 8)
        # columns of the attention's input gradient in the backward: q | k | v [| R, 10 rows per head, clipped_causal], padded to 8
        self.kcat = (3 * hidsize + NBASIS * attention_heads + 7) // 8 * 8 if self.mask_style == "clipped_causal" else 3 * hidsize

    def forward_flops_per_frame(self, head_outputs: int = 121 + 8641 + 1) -> float:
        """Algorithmic work of one frame through the forward path (SURVEY.md section 8d): 2 x MAC; clipped-causal attention counts
        `maxlen` keys per query (the band), unmasked attention (IDM) every key of the chunk.  bench.py's roofline uses this."""
        H, W = self.img_shape[0], self.img_shape[1]
        fl, cin = 0.0, 3
        if self.conv3d_out is not None:
            fl += 2 * H * W * 15 * self.conv3d_out
            cin = self.conv3d_out
        for c in self.chans:
            fl += 2 * H * W * 9 * cin * c
            H, W = (H + 1) // 2, (W + 1) // 2
            fl += 4 * 2 * H * W * 9 * c * c
            cin = c
        h = self.hidsize
        fl += 2 * (cin * H * W) * self.cnn_outsize + 2 * self.cnn_outsize * h
        keys = self.maxlen if self.mask_style == "clipped_causal" else self.maxlen + (self.timesteps or 0)
        nb = NBASIS if self.mask_style == "clipped_causal" else 0
        per_layer = 2 * h * h * 4 + 2 * h * nb * self.heads + 2 * 2 * h * h * self.pointwise_ratio
        per_layer += 4 * keys * h + 2 * nb * keys * self.heads
        fl += self.n_layers * per_layer + (2 * h * h if self.conv3d_out is None else 0) + 2 * h * head_outputs
        return fl


def _net_schema(cfg: NetConfig) -> "OrderedDict[str, torch.Tensor]":
    """Freshly initialised parameters in the reference's registration order (lib/impala_cnn.py, lib/util.py, lib/xf.py)."""
    sd = OrderedDict()
    p = "img_process.cnn"
    cin = cfg.img_shape[2]
    nstack = len(cfg.chans)
    for i, c in enumerate(cfg.chans):
        s = f"{p}.stacks.{i}"
        has_norm = cfg.first_conv_norm if i == 0 else True
        if has_norm:
            sd[f"{s}.firstconv.norm.weight"], sd[f"{s}.firstconv.norm.bias"] = torch.ones(cin), torch.zeros(cin)
        sd[f"{s}.firstconv.layer.weight"] = _fanin((c, cin, 3, 3), 1.0)
        if not has_norm:
            sd[f"{s}.firstconv.layer.bias"] = torch.zeros(c)
        sd[f"{s}.n.weight"], sd[f"{s}.n.bias"] = torch.ones(c), torch.zeros(c)
        bs = math.sqrt(math.sqrt(nstack) / math.sqrt(2))  # impala_cnn.py:164,105,30
        for j in range(2):
            for k in range(2):
                q = f"{s}.blocks.{j}.conv{k}"
                sd[f"{q}.norm.weight"], sd[f"{q}.norm.bias"] = torch.ones(c), torch.zeros(c)
                sd[f"{q}.layer.weight"] = _fanin((c, c, 3, 3), bs)
        cin = c
    kd = cin * cfg.final_hw[0] * cfg.final_hw[1]
    sd[f"{p}.dense.norm.weight"], sd[f"{p}.dense.norm.bias"] = torch.ones(kd), torch.zeros(kd)
    sd[f"{p}.dense.layer.weight"] = _fanin((cfg.cnn_outsize, kd), 1.4)
    sd["img_process.linear.norm.weight"], sd["img_process.linear.norm.bias"] = torch.ones(256), torch.zeros(256)
    sd["img_process.linear.layer.weight"] = _fanin((cfg.hidsize, 256), 1.0)
    h = cfg.hidsize
    s_blk = cfg.n_layers ** -0.5 * 2 ** -0.5  # lib/util.py:101,154-155
    s_att = math.sqrt(s_blk)                  # lib/xf.py:246
    for l in range(cfg.n_layers):
        b = f"recurrent_layer.blocks.{l}"
        sd[f"{b}.mlp0.norm.weight"], sd[f"{b}.mlp0.norm.bias"] = torch.ones(h), torch.zeros(h)
        sd[f"{b}.mlp0.layer.weight"] = _fanin((h * cfg.pointwise_ratio, h), 1.0)
        sd[f"{b}.mlp1.layer.weight"] = _fanin((h, h * cfg.pointwise_ratio), s_blk)
        sd[f"{b}.mlp1.layer.bias"] = torch.zeros(h)
        sd[f"{b}.pre_r_ln.weight"], sd[f"{b}.pre_r_ln.bias"] = torch.ones(h), torch.zeros(h)
        o = f"{b}.r.orc_block"
        sd[f"{o}.b_nd"] = torch.randn(NBASIS, cfg.maxlen) * 0.2
        sd[f"{o}.q_layer.weight"], sd[f"{o}.q_layer.bias"] = _fanin((h, h), 0.1), torch.zeros(h)
        sd[f"{o}.k_layer.weight"] = _fanin((h, h), 0.2)
        sd[f"{o}.v_layer.weight"] = _fanin((h, h), 1.0 * s_att)
        sd[f"{o}.proj_layer.weight"], sd[f"{o}.proj_layer.bias"] = _fanin((h, h), 1.0 * s_att), torch.zeros(h)
        sd[f"{o}.r_layer.weight"], sd[f"{o}.r_layer.bias"] = _fanin((NBASIS * cfg.heads, h), 0.1), torch.zeros(NBASIS * cfg.heads)
    sd["lastlayer.norm.weight"], sd["lastlayer.norm.bias"] = torch.ones(h), torch.zeros(h)
    sd["lastlayer.layer.weight"] = _fanin((h, h), 1.0)
    sd["final_ln.weight"], sd["final_ln.bias"] = torch.ones(h), torch.zeros(h)
    if cfg.conv3d_out is not None:  # lib/policy.py:362-372 (registered after the base class's modules)
        sd["conv3d_layer.layer.weight"] = _fanin((cfg.conv3d_out, 3, 5, 1, 1), 1.0)
        sd["conv3d_layer.layer.bias"] = torch.zeros(cfg.conv3d_out)
    return sd


# ---------------------------------------------------------------------------------------------------------------
# kernel-side weight layouts
# ---------------------------------------------------------------------------------------------------------------
_CLASS_TAPS = None


def _class_taps(device):
    """[9 border classes][9 taps] 0/1 matrix (float64): which taps of a 3x3 pad-1 convolution read inside the image for an output
    pixel of border class (cy, cx), cy / cx in {first row / column, interior, last row / column}."""
    global _CLASS_TAPS
    if _CLASS_TAPS is None or _CLASS_TAPS.device != device:
        valid = {0: [1, 2], 1: [0, 1, 2], 2: [0, 1]}
        m = torch.zeros(9, 9, dtype=torch.float64)
        for cy in range(3):
            for cx in range(3):
                for ky in valid[cy]:
                    for kx in valid[cx]:
                        m[cy * 3 + cx, ky * 3 + kx] = 1.0
        _CLASS_TAPS = m.to(device)
    return _CLASS_TAPS


def _fold_conv(W, gamma, beta):
    """GroupNorm(1) -> conv3x3(pad 1) fold (SURVEY.md section 7.2):
    conv(GN(x))[o,p] = rstd*conv_{W*gamma}(x)[o,p] - rstd*mean*S1[cls(p)][o] + S2[cls(p)][o].
    S1 is summed from the bf16-ROUNDED weights (the ones the tensor cores multiply) so the mean term cancels exactly.
    (Runs after every optimizer step of a BC run, hence a handful of batched ops rather than a loop over the 9 classes.)"""
    Cout = W.shape[0]
    Wg = (W * gamma[None, :, None, None]).permute(0, 2, 3, 1).contiguous()  # [Cout, ky, kx, Cin]
    Wb = Wg.to(BF16)
    tg = Wb.sum(-1, dtype=torch.float64).reshape(Cout, 9)                                  # per-tap sums of W*gamma
    tb = (W * beta[None, :, None, None]).sum(1, dtype=torch.float64).reshape(Cout, 9)      # per-tap sums of W*beta
    M = _class_taps(W.device)
    S1 = (M @ tg.t()).float().contiguous()  # [9, Cout]
    S2 = (M @ tb.t()).float().contiguous()
    return Wb.reshape(Cout, -1).contiguous(), S1, S2


def _fold_conv2(W, gamma0, beta0, gamma_n, beta_n):
    """Two-norm composition for block 0's conv0 (x0 = GN_n(y1) is not materialised; the conv reads y1):
    conv(GN_0(GN_n(y1))) = R * conv_{W g0 gn}(y1) + rstd0*Ta - R*mu1*Tb - rstd0*mu0*Tc + Td   per border class (see vpt_norm2_fold).
    Returns (bf16 weights [Cout, 9*Cin], (Ta, Tb, Tc, Td) fp32 [9, Cout]); Tb is summed from the bf16-rounded weights."""
    Cout = W.shape[0]
    Wb = (W * (gamma0 * gamma_n)[None, :, None, None]).permute(0, 2, 3, 1).contiguous().to(BF16)  # [Cout, ky, kx, Cin]
    M = _class_taps(W.device)
    per_tap = lambda v: v.reshape(Cout, 9)
    tb = per_tap(Wb.sum(-1, dtype=torch.float64))
    ta = per_tap((W * (gamma0 * beta_n)[None, :, None, None]).sum(1, dtype=torch.float64))
    tc = per_tap((W * gamma0[None, :, None, None]).sum(1, dtype=torch.float64))
    td = per_tap((W * beta0[None, :, None, None]).sum(1, dtype=torch.float64))
    tabs = tuple((M @ t.t()).float().contiguous() for t in (ta, tb, tc, td))
    return Wb.reshape(Cout, -1).contiguous(), tabs


def _fold_linear(W, gamma=None, beta=None, bias=None):
    """[LayerNorm ->] Linear fold: out = rstd*(x @ (W*gamma)^T) - rstd*mean*S1 + S2, S2 = W @ beta (+ bias)."""
    Wg = W if gamma is None else W * gamma[None, :]
    Wb = Wg.to(BF16).contiguous()
    S1 = Wb.sum(1, dtype=torch.float64).float().contiguous() if gamma is not None else None
    S2 = None
    if beta is not None:
        S2 = (W * beta[None, :]).sum(1, dtype=torch.float64)
    if bias is not None:
        S2 = bias.double() if S2 is None else S2 + bias.double()
    return Wb, S1, (S2.float().contiguous() if S2 is not None else None)


def _dense_to_zp(v, cfg: NetConfig):
    """The `dense` layer's input dimension (last axis of `v`): the reference flatten order c*H*W + h*W + w (lib/impala_cnn.py:192-193)
    -> our ZP layout [Hf+1][Wf+1][C2], i.e. (h, w, c) order with zero columns where the layout holds its zero row / column."""
    Hf, Wf = cfg.final_hw
    v = v.reshape(*v.shape[:-1], cfg.chans[-1], Hf, Wf).movedim(-3, -1)  # (..., Hf, Wf, C2)
    v = torch.nn.functional.pad(v, (0, 0, 0, 1, 0, 1))                     # (..., Hf+1, Wf+1, C2)
    return v.reshape(*v.shape[:-3], -1)


def _dense_from_zp(v, cfg: NetConfig):
    """Inverse of `_dense_to_zp`: ZP (h, w, c) order -> the reference C,H,W flatten order, dropping the pad row / column."""
    Hf, Wf = cfg.final_hw
    v = v.reshape(*v.shape[:-1], Hf + 1, Wf + 1, cfg.chans[-1])[..., :Hf, :Wf, :]
    return v.movedim(-1, -3).reshape(*v.shape[:-3], -1)


def _rot(W):
    """conv weight [Cout, Cin, 3, 3] -> dgrad weight bf16 [Cin][tap'][Cout] with tap' = 8 - tap (180-degree rotation)."""
    return W.detach().flip(2, 3).permute(1, 2, 3, 0).reshape(W.shape[1], -1).to(BF16).contiguous()


def _tr(W, pad_to=None):
    """linear weight [out, in] -> dgrad weight bf16 [in][out] (optionally zero-padded along `out` to `pad_to` columns)."""
    Wt = W.detach().t().to(BF16)
    if pad_to is not None and pad_to != Wt.shape[1]:
        Wt = torch.nn.functional.pad(Wt, (0, pad_to - Wt.shape[1]))
    return Wt.contiguous()


class _Prepared:
    """Device-side, kernel-layout copy of the parameters of one MinecraftPolicy (+ optional heads)."""

    def __init__(self, cfg: NetConfig, sd: Dict[str, torch.Tensor], prefix: str = ""):
        g = lambda k: sd[prefix + k].detach()
        p = "img_process.cnn"
        self.conv3d = None
        if cfg.conv3d_out is not None:  # [C, 3, dt, 1, 1] -> [C][dt][c] / 255
            w3 = g("conv3d_layer.layer.weight").double().reshape(cfg.conv3d_out, 3, 5).permute(0, 2, 1).reshape(cfg.conv3d_out, 15) / 255.0
            self.conv3d = (w3.float().contiguous(), g("conv3d_layer.layer.bias").float().contiguous())
        self.stacks = []
        for i, c in enumerate(cfg.chans):
            s = f"{p}.stacks.{i}"
            st = {}
            if i == 0 and not cfg.first_conv_norm:
                w = g(f"{s}.firstconv.layer.weight")  # [C0, 3, ky, kx] -> [C0][ky][kx][c] / 255 (lib/policy.py:44)
                st["fc_w"] = (w.double().permute(0, 2, 3, 1).reshape(c, 27) / 255.0).float().contiguous()
                st["fc_b"] = g(f"{s}.firstconv.layer.bias").float().contiguous()
            else:
                st["first"] = _fold_conv(g(f"{s}.firstconv.layer.weight"), g(f"{s}.firstconv.norm.weight"), g(f"{s}.firstconv.norm.bias"))
            st["n_g"], st["n_b"] = g(f"{s}.n.weight").float().contiguous(), g(f"{s}.n.bias").float().contiguous()
            q0 = f"{s}.blocks.0.conv0"
            st["conv0n"] = _fold_conv2(g(f"{q0}.layer.weight"), g(f"{q0}.norm.weight"), g(f"{q0}.norm.bias"), g(f"{s}.n.weight"), g(f"{s}.n.bias"))
            st["convs"] = []
            for j in range(2):
                for k in range(2):
                    q = f"{s}.blocks.{j}.conv{k}"
                    st["convs"].append(_fold_conv(g(f"{q}.layer.weight"), g(f"{q}.norm.weight"), g(f"{q}.norm.bias")))
            self.stacks.append(st)
        perm = lambda v: _dense_to_zp(v, cfg)
        self.dense = _fold_linear(perm(g(f"{p}.dense.layer.weight")), perm(g(f"{p}.dense.norm.weight")), perm(g(f"{p}.dense.norm.bias")))
        self.linear = _fold_linear(g("img_process.linear.layer.weight"), g("img_process.linear.norm.weight"), g("img_process.linear.norm.bias"))
        self.layers = []
        for l in range(cfg.n_layers):
            b = f"recurrent_layer.blocks.{l}"
            o = f"{b}.r.orc_block"
            L = {}
            L["ln_g"], L["ln_b"] = g(f"{b}.pre_r_ln.weight").float().contiguous(), g(f"{b}.pre_r_ln.bias").float().contiguous()
            L["q"] = _fold_linear(g(f"{o}.q_layer.weight"), bias=g(f"{o}.q_layer.bias"))
            L["k"] = _fold_linear(g(f"{o}.k_layer.weight"))
            L["v"] = _fold_linear(g(f"{o}.v_layer.weight"))
            L["r"] = _fold_linear(g(f"{o}.r_layer.weight"), bias=g(f"{o}.r_layer.bias"))
            # fused projection (lib/xf.py:334-365: Q(+bias) | K | V | R(+bias) of the same x_hat): one GEMM over the concatenated weight with
            # four column segments, each with its own destination (csrc/gemm_tc.cuh, vpt_gemm_args.dst_*)
            causal = cfg.mask_style == "clipped_causal"
            ws = [g(f"{o}.q_layer.weight"), g(f"{o}.k_layer.weight"), g(f"{o}.v_layer.weight")] + ([g(f"{o}.r_layer.weight")] if causal else [])
            zb = torch.zeros_like(g(f"{o}.q_layer.bias"))
            bs = [g(f"{o}.q_layer.bias"), zb, zb] + ([g(f"{o}.r_layer.bias")] if causal else [])
            L["qkvr"] = _fold_linear(torch.cat(ws, 0), bias=torch.cat(bs, 0))
            L["b_nd"] = g(f"{o}.b_nd").float().contiguous()
            L["proj"] = _fold_linear(g(f"{o}.proj_layer.weight"), bias=g(f"{o}.proj_layer.bias"))
            L["mlp0"] = _fold_linear(g(f"{b}.mlp0.layer.weight"), g(f"{b}.mlp0.norm.weight"), g(f"{b}.mlp0.norm.bias"))
            L["mlp1"] = _fold_linear(g(f"{b}.mlp1.layer.weight"), bias=g(f"{b}.mlp1.layer.bias"))
            self.layers.append(L)
        self.last = _fold_linear(g("lastlayer.layer.weight"), g("lastlayer.norm.weight"), g("lastlayer.norm.bias"))
        self.fin_g, self.fin_b = g("final_ln.weight").float().contiguous(), g("final_ln.bias").float().contiguous()


def _fingerprint(params):
    return tuple((p.data_ptr(), p._version) for p in params)


class _Versioned:
    """One kernel-layout copy of some parameters and the versions it was made from: `get()` rebuilds it when a parameter has new storage
    (a load, `.to()`) or was updated in place (an optimizer step; FlatAdamDP bumps `_version` after its kernel writes).  `params` and
    `build` are bound methods of the owning module, so that a deep copy of the module owns its own copy; `build` makes weights only,
    since `_PolicyBase.refresh_weights` also runs it inside a CUDA graph capture."""

    def __init__(self, params, build):
        self.params, self.build = params, build
        self.fp = self.value = None

    def stale(self):
        return self.value is None or _fingerprint(self.params()) != self.fp

    def get(self):
        if self.stale():
            with torch.no_grad():
                self.set(self.build())
        return self.value

    def set(self, value):
        self.value, self.fp = value, _fingerprint(self.params())


def _differentiable(module: nn.Module, img=None) -> bool:
    """The forward builds an autograd graph only when asked to (`set_autograd`), in grad mode outside inference mode, and when at least
    one parameter or the image `img` requires grad; otherwise the inference path runs, bit for bit."""
    return module._autograd and torch.is_grad_enabled() and not torch.is_inference_mode_enabled() and \
        ((img is not None and img.requires_grad) or any(p.requires_grad for p in module.parameters()))


def frames_f32(img):
    """lib/policy.py:39-45 takes any frames `img.to(float32)` converts: uint8 frames stay uint8 (the kernels' u8 path), a floating
    dtype (values on the uint8 scale, not clipped) becomes fp32 here, so that autograd carries the gradient of a float16 / bfloat16 /
    float64 leaf back in its own dtype.  Other integer dtypes raise TypeError."""
    if img.dtype == torch.uint8:
        return img
    if not img.dtype.is_floating_point:
        raise TypeError(f"ob['img'] must be uint8 or a floating dtype on the uint8 scale (B,T,H,W,3) as in the reference (lib/policy.py:39-45); "
                        f"got {img.dtype}")
    return img.to(torch.float32)


LATENT_KEY = "img_latent"  # the observation key of cached CNN latents: policy({"img_latent": lat}, first, state)
CNN_PREFIXES = ("img_process.cnn.", "conv3d_layer.")  # the network's parameters at or below the `dense` layer: the CNN part


class FrameLatents:
    """The output of the CNN part of a network (`MinecraftPolicy.encode`): per frame the `dense` layer's output `x`, bf16 (..., 256), and
    its row statistics `stats`, fp32 (..., 2) (mean, rstd from the dense GEMM's epilogue, which `img_process.linear`'s folded LayerNorm
    reads), over the leading dimensions (B, T).  `token` identifies the encoding network's CNN weights (`MinecraftPolicy.check_latents`).

    Only what a data loader needs: indexing over the leading dimensions, `FrameLatents.cat(list, dim)` and `.to(device)`.  Latents carry
    no autograd graph and cannot require grad.  The IDM's latents hold its conv3d pre-stage, which mixes five neighbouring frames of a
    sequence: they stay valid when re-batched along B, not when sliced along T."""

    def __init__(self, x, stats, token=None):
        if x.requires_grad or stats.requires_grad:
            raise ValueError("FrameLatents carry no autograd graph: x and stats must not require grad")
        if tuple(stats.shape) != (*x.shape[:-1], 2):
            raise ValueError(f"FrameLatents: stats {tuple(stats.shape)} must be x's leading shape {tuple(x.shape[:-1])} + (2,)")
        self.x, self.stats, self.token = x, stats, token

    @property
    def shape(self):
        """The leading (frame) dimensions, (B, T) for a forward's input."""
        return self.x.shape[:-1]

    @property
    def device(self):
        return self.x.device

    @property
    def requires_grad(self):
        return self.x.requires_grad or self.stats.requires_grad

    def __getitem__(self, idx):
        parts = idx if isinstance(idx, tuple) else (idx,)
        used = sum(0 if p is None else p.dim() if isinstance(p, torch.Tensor) and p.dtype == torch.bool else 1 for p in parts)
        if any(p is Ellipsis for p in parts) or used > self.x.dim() - 1:
            raise IndexError(f"FrameLatents index only the leading {self.x.dim() - 1} dimension(s), without Ellipsis")
        return FrameLatents(self.x[idx], self.stats[idx], self.token)

    @staticmethod
    def cat(latents, dim=0):
        """torch.cat over a leading dimension of latents encoded with the same CNN weights."""
        latents = list(latents)
        lead = latents[0].x.dim() - 1
        if not -lead <= dim < lead:
            raise IndexError(f"FrameLatents.cat: dim {dim} is not one of the {lead} leading dimension(s)")
        dim %= lead
        if any(lat.token != latents[0].token for lat in latents[1:]):
            raise ValueError("FrameLatents.cat: the latents were encoded with different CNN weights")
        return FrameLatents(torch.cat([lat.x for lat in latents], dim), torch.cat([lat.stats for lat in latents], dim), latents[0].token)

    def to(self, device, non_blocking=False):
        return FrameLatents(self.x.to(device, non_blocking=non_blocking), self.stats.to(device, non_blocking=non_blocking), self.token)


class RingState:
    """The recurrent state of `MinecraftAgentPolicy` as a ring that a t = 1 forward (`act`, `v`, `get_output_for_observation`, `forward`,
    `GraphedAct(memory="ring")`) updates in place, instead of building a new state from a copy of the old one.  Per layer the KV memory
    K / V is bf16 (B, maxlen, h) and the state mask bool (B, maxlen); memory row j (oldest first) is at physical row (off + j) % maxlen,
    where `off` is one device int32 shared by the layers.  A step writes its K / V rows at `off`, attends, and advances `off`: nothing else
    of the memory moves.  The step's results are those of the same step from `to_pytree()`, bit for bit: the pytree path rounds its fp32
    state to bf16 before the attention reads it, and every row it stores came out of a bf16 GEMM.

    The forward returns the RingState it was given, updated: copy it out with `to_pytree()` first to keep the old state.

    Asynchronous rollouts step some of the ring's environments at a time through a view, `ring.rows(idx)` (`RingRows`).  They need one
    offset per environment: `row_off`, None (all zeros) until the first call that needs it allocates a device int32 (E,); memory row j of
    environment e is then at physical row (off + row_off[e] + j) % maxlen.  A step of the whole ring advances `off`, a step of a view
    advances `row_off` of the rows it stepped.

    In the batch-invariant mode (`MinecraftAgentPolicy.set_batch_invariant`) `act` samples environment e's step with the noise key
    (stream e, step steps[e]): `steps` is None until the first such `act` allocates a device int64 (E,) of zeros, and each such `act`
    advances it, on the device, for the environments it stepped (never for an inert row).  `to_pytree` / `load_` leave it alone; set it in
    place (`ring.steps[e] = s`) to replay environment e from its step s."""

    def __init__(self, k, v, mask, off, row_off=None):
        self.k, self.v, self.mask, self.off = k, v, mask, off  # per layer: bf16 (E, maxlen, h) x 2, bool (E, maxlen); int32 (1,)
        self.row_off = row_off  # None or int32 (E,), each in [0, maxlen)
        self.steps = None  # None or int64 (E,): the batch-invariant mode's per-environment sampling step

    @staticmethod
    def _net(policy):
        net = getattr(policy, "net", policy)
        if isinstance(net, InverseActionNet):
            raise TypeError("the IDM has no KV memory across calls: RingState is for MinecraftAgentPolicy / MinecraftPolicy")
        if not isinstance(net, MinecraftPolicy):
            raise TypeError(f"RingState: expected a MinecraftAgentPolicy or MinecraftPolicy, got {type(policy).__name__}")
        if net.cfg.maxlen == 0 or net.cfg.mask_style != "clipped_causal":
            raise ValueError("RingState needs a KV memory: attention_memory_size > timesteps with the clipped_causal mask")
        return net

    @classmethod
    def zeros(cls, policy, B: int) -> "RingState":
        """The state of `policy.initial_state(B)` (empty memory, every mask bit clear) on the policy's device."""
        net = cls._net(policy)
        cfg, dev = net.cfg, net.final_ln.weight.device
        L, maxlen, h = cfg.n_layers, cfg.maxlen, cfg.hidsize
        k = torch.zeros((L, B, maxlen, h), dtype=BF16, device=dev)
        v = torch.zeros((L, B, maxlen, h), dtype=BF16, device=dev)
        mask = torch.zeros((L, B, maxlen), dtype=torch.bool, device=dev)
        return cls(list(k.unbind(0)), list(v.unbind(0)), list(mask.unbind(0)), torch.zeros((1,), dtype=torch.int32, device=dev))

    @classmethod
    def from_pytree(cls, policy, state) -> "RingState":
        """A ring holding the reference-format state `state` (`initial_state` / a `state_out`: per layer (mask (B, 1, maxlen) or None,
        (K, V) (B, maxlen, h))); fp32 K / V are rounded to bf16 by the kernel, and so exactly as, the pytree forward rounds them."""
        cls._net(policy)
        ring = cls.zeros(policy, state[0][1][0].shape[0])
        ring.load_(state)
        return ring

    @property
    def batch_size(self):
        return self.k[0].shape[0]

    def _alloc_row_off(self):
        if self.row_off is None:
            self.row_off = torch.zeros((self.batch_size,), dtype=torch.int32, device=self.off.device)
        return self.row_off

    def _alloc_steps(self):
        if self.steps is None:
            self.steps = torch.zeros((self.batch_size,), dtype=torch.int64, device=self.off.device)
        return self.steps

    def rows(self, idx) -> "RingRows":
        """A view of the environments `idx` (a 1-D integer sequence, CPU or CUDA tensor) for a t = 1 step of those only: row i of the
        call's obs and `first` is environment idx[i]'s next frame, and -1 marks an inert padding row.  Validated here, on the host (a CUDA
        `idx` is copied back once); raises ValueError for an entry outside [-1, E) or an environment listed twice."""
        host = idx.detach().to("cpu") if torch.is_tensor(idx) else torch.as_tensor(idx)
        if host.dim() != 1 or host.numel() == 0 or host.dtype.is_floating_point or host.dtype.is_complex or host.dtype == torch.bool:
            raise ValueError(f"RingState.rows: idx must be a non-empty 1-D integer sequence (got {host.dtype} {tuple(host.shape)})")
        E = self.batch_size
        envs = host.tolist()
        bad = [e for e in envs if not -1 <= e < E]
        if bad:
            raise ValueError(f"RingState.rows: rows {bad} are outside the ring's {E} environments (or -1 for padding)")
        real = [e for e in envs if e >= 0]
        if len(set(real)) != len(real):
            raise ValueError(f"RingState.rows: an environment is listed twice in {envs}")
        return RingRows(self, torch.tensor(envs, dtype=torch.int32).to(self.off.device, non_blocking=True), envs)

    def load_(self, state):
        """Copy `state` (a pytree as in `from_pytree`, or a RingState of the same shape) into this ring, in place.  A pytree is written at
        rotation 0 (`row_off` zeroed); a ring's `row_off` is copied."""
        L, (B, maxlen, h) = len(self.k), self.k[0].shape
        if isinstance(state, RingRows):
            raise ValueError("RingState.load_: a view of a ring; load its `to_pytree()`, or use `view.load_` to write into a view")
        if isinstance(state, RingState):
            if len(state.k) != L or state.k[0].shape != self.k[0].shape:
                raise ValueError(f"RingState.load_: a ring of {len(state.k)} x {tuple(state.k[0].shape)} into one of {L} x {(B, maxlen, h)}")
            for dst, src in zip(self.k + self.v + self.mask + [self.off], state.k + state.v + state.mask + [state.off]):
                dst.copy_(src)
            if state.row_off is not None:
                self._alloc_row_off().copy_(state.row_off)
            elif self.row_off is not None:
                self.row_off.zero_()
            return self
        if len(state) != L:
            raise ValueError(f"RingState.load_: a state of {len(state)} layers into a ring of {L}")
        for l, (m, (K, V)) in enumerate(state):
            if tuple(K.shape) != (B, maxlen, h) or V.shape != K.shape:
                raise ValueError(f"RingState.load_: layer {l} K / V {tuple(K.shape)} / {tuple(V.shape)} != {(B, maxlen, h)}")
            if K.dtype not in (F32, BF16) or V.dtype not in (F32, BF16):
                raise TypeError(f"RingState.load_: K / V must be float32 or bfloat16 (got {K.dtype}, {V.dtype})")
            if m is None:
                self.mask[l].zero_()  # lib/masked_attention.py:75-76: None == all-False
            else:
                self.mask[l].copy_(m.reshape(B, maxlen))
            if K.stride() == V.stride() and K.dtype == V.dtype:
                ops.copy_rows2(K, V, 0, self.k[l], self.v[l], 0, maxlen)
            else:
                ops.copy_rows(K, 0, self.k[l], 0, maxlen)
                ops.copy_rows(V, 0, self.v[l], 0, maxlen)
        self.off.zero_()
        if self.row_off is not None:
            self.row_off.zero_()
        return self

    def _gather(self, sel):
        """The reference-format state of the ring rows `sel` (a device int64 vector), each rotated by its own offset (bf16 -> fp32 is exact)."""
        maxlen, h = self.k[0].shape[1:]
        shift = self.off if self.row_off is None else self.off + self.row_off[sel]
        phys = ((shift.long()[:, None] + torch.arange(maxlen, device=sel.device)) % maxlen).expand(sel.numel(), maxlen)
        idx = phys[:, :, None].expand(-1, -1, h)
        out = []
        for k, v, m in zip(self.k, self.v, self.mask):
            K = k.index_select(0, sel).gather(1, idx).float()
            V = v.index_select(0, sel).gather(1, idx).float()
            out.append((m.index_select(0, sel).gather(1, phys).unsqueeze(1), (K, V)))
        return out

    def to_pytree(self):
        """The reference-format state, a new list[(mask bool (B, 1, maxlen), (K, V) fp32 (B, maxlen, h))] with the oldest row first; after
        a step it is the pytree forward's `state_out`, bit for bit.  Reads `off` back to the host (synchronises) unless `row_off` is
        allocated: each environment is then rotated by its own offset on the device."""
        B, maxlen, h = self.k[0].shape
        if self.row_off is not None:
            return self._gather(torch.arange(B, device=self.off.device))
        off = int(self.off.item())
        out = []
        for k, v, m in zip(self.k, self.v, self.mask):
            K = torch.empty((B, maxlen, h), dtype=F32, device=k.device)
            V = torch.empty_like(K)
            ops.copy_rows2(k, v, off, K, V, 0, maxlen - off)
            ops.copy_rows2(k, v, 0, K, V, maxlen - off, off)
            out.append((torch.cat([m[:, off:], m[:, :off]], 1).unsqueeze(1), (K, V)))
        return out


class RingRows:
    """A view of some environments of a `RingState` (`ring.rows(idx)`), accepted wherever a RingState is: a t = 1 step of environments
    idx[0], idx[1], ... (row i of obs and `first`), which updates their memory and their `row_off` in place and returns the same view.
    Every other environment is untouched.  A -1 entry is an inert padding row: it reads and writes no ring memory, its attention output
    is zero, and its outputs (actions, log-probs, vpred, pd) are finite and meaningless.

    `idx` is a device int32 copy of the environments (`envs`, host ints); `GraphedAct(..., envs=E)` replays one graph over its own views."""

    def __init__(self, ring: RingState, idx, envs):
        self.ring, self.idx, self.envs = ring, idx, envs

    def __len__(self):
        return len(self.envs)

    @property
    def batch_size(self):
        return len(self.envs)

    def _sel(self, what):
        if any(e < 0 for e in self.envs):
            raise ValueError(f"RingRows.{what}: the view has inert (-1) rows")
        return self.idx.long()

    def to_pytree(self):
        """The listed environments' reference-format state, in `idx` order (as `RingState.to_pytree`; no -1 entry)."""
        return self.ring._gather(self._sel("to_pytree"))

    def load_(self, state):
        """Write `state`, a reference-format state of len(idx) rows, into the listed environments only (no -1 entry).  Each is stored at
        rotation 0 with row_off[e] = -off mod maxlen; fp32 K / V are rounded to bf16 as the pytree forward rounds them."""
        ring = self.ring
        sel = self._sel("load_")
        L, (E, maxlen, h) = len(ring.k), ring.k[0].shape
        n = len(self)
        if isinstance(state, (RingState, RingRows)):
            raise ValueError("RingRows.load_ takes a reference-format state (a ring's `to_pytree()`)")
        if len(state) != L:
            raise ValueError(f"RingRows.load_: a state of {len(state)} layers into a ring of {L}")
        for l, (m, (K, V)) in enumerate(state):
            if tuple(K.shape) != (n, maxlen, h) or V.shape != K.shape:
                raise ValueError(f"RingRows.load_: layer {l} K / V {tuple(K.shape)} / {tuple(V.shape)} != {(n, maxlen, h)}")
            if K.dtype not in (F32, BF16) or V.dtype not in (F32, BF16):
                raise TypeError(f"RingRows.load_: K / V must be float32 or bfloat16 (got {K.dtype}, {V.dtype})")
        for l, (m, (K, V)) in enumerate(state):
            ring.k[l].index_copy_(0, sel, K.to(device=sel.device, dtype=BF16))
            ring.v[l].index_copy_(0, sel, V.to(device=sel.device, dtype=BF16))
            if m is None:
                ring.mask[l].index_fill_(0, sel, False)  # lib/masked_attention.py:75-76: None == all-False
            else:
                ring.mask[l].index_copy_(0, sel, m.reshape(n, maxlen).to(device=sel.device, dtype=torch.bool))
        rot0 = ((maxlen - ring.off) % maxlen).to(torch.int32)  # off + row_off[e] = 0 (mod maxlen): memory row j at physical row j
        ring._alloc_row_off().index_copy_(0, sel, rot0.expand(n).contiguous())
        return self


_RING_STATES = (RingState, RingRows)


def _check_ring_call(net, img, state_in, differentiable: bool):
    """Raises, before any launch, for a forward call a RingState (or a view of one) cannot serve."""
    RingState._net(net)
    if net.precision != "bf16":
        raise NotImplementedError("RingState runs in the bf16 mode only (set_precision('bf16'))")
    if differentiable or net._tape is not None:
        raise ValueError("RingState is for inference: the differentiable forward and the trainers take the pytree state")
    B, t = img.shape[:2]
    if t != 1:
        raise ValueError(f"RingState takes one frame per call (t = 1, got t = {t}): a chunk's rows would overwrite memory that its "
                         "earlier frames still attend to")
    ring, E = state_in, B
    if isinstance(state_in, RingRows):
        if len(state_in) != B:
            raise ValueError(f"a view of {len(state_in)} ring rows for a call of B = {B}")
        ring = state_in.ring
        E = ring.batch_size
    cfg = net.cfg
    if len(ring.k) != cfg.n_layers or tuple(ring.k[0].shape) != (E, cfg.maxlen, cfg.hidsize):
        raise ValueError(f"RingState of {len(ring.k)} x {tuple(ring.k[0].shape)} for a call of {cfg.n_layers} x "
                         f"{(E, cfg.maxlen, cfg.hidsize)}")


def _ob_input(ob):
    """The network input of an observation dict: the frames `ob["img"]` or the latents `ob["img_latent"]` (exactly one of them)."""
    if LATENT_KEY not in ob:
        return ob["img"]
    if "img" in ob:
        raise ValueError(f"the observation holds both 'img' and {LATENT_KEY!r}: pass one of them")
    lat = ob[LATENT_KEY]
    if not isinstance(lat, FrameLatents):
        raise TypeError(f"ob[{LATENT_KEY!r}] must be FrameLatents (from encode), got {type(lat).__name__}")
    return lat


def _add_time(v):
    """(B, ...) -> (B, 1, ...) for frames or latents (get_output_for_observation)."""
    return v[:, None] if isinstance(v, FrameLatents) else v.unsqueeze(1)


def check_recompute_frames(v):
    """`recompute_frames` of the trainers and `set_autograd`: None (keep the CNN's activations for the backward) or a positive int."""
    if v is not None and (isinstance(v, bool) or not isinstance(v, int) or v <= 0):
        raise ValueError(f"recompute_frames must be None or a positive int (got {v!r})")
    return v


def _autograd_runner(module: nn.Module):
    """The module's differentiable-forward machinery (training._AutogradRunner), made on first use.  Tests read the tape of the last
    differentiable call from it (`keep_tape` / `last_tape`, as with the trainers)."""
    if module._ag_runner is None:
        from .training import _AutogradRunner
        module._ag_runner = _AutogradRunner(module)
    return module._ag_runner


# ---------------------------------------------------------------------------------------------------------------
# MinecraftPolicy
# ---------------------------------------------------------------------------------------------------------------
class MinecraftPolicy(nn.Module):
    """lib/policy.py:83-224.  `forward(ob, state_in, context)` -> ((pi_latent, vf_latent), state_out)."""

    cnn_chunk_frames = 2048  # frames per CNN pass (bounds the activation workspace: ~5 MiB/frame at 2x width)
    fold_stack_norm = True   # inference: fold the post-pool GroupNorm of every stack into block 0 (no `affine_norm_zp` pass)
    idm_chunk_frames = 512   # IDM: ~13 MiB/frame at 4x width (conv3d output + full-resolution first conv)
    use_lastlayer = True     # the forward runs `lastlayer` between the transformer and final_ln

    def __init__(self, **policy_kwargs):
        super().__init__()
        self.cfg = NetConfig(**policy_kwargs)
        self.hidsize = self.cfg.hidsize
        self.single_output = self.cfg.single_output
        for name, t in _net_schema(self.cfg).items():
            _set(self, name, t)
        self._fold = _Versioned(self.parameters, self._build_prepared)
        self._fold_fp32 = _Versioned(self.parameters, self._build_prepared_precise)
        self._bwd = _Versioned(self.parameters, self._build_backward)
        self.precision = "bf16"  # "fp32": the fp32-parity mode (precise.py): bf16 hi/lo split operands, fp32 activations
        self.debug_taps = None  # set to a dict to capture intermediate activations (tests)
        self._tape = None       # set to a dict by training.BCTrainer: the forward then records what the backward needs
        self._autograd = False  # set_autograd
        self._state_grad = False
        self._recompute_frames = None
        self._ag_runner = None

    def output_latent_size(self):
        return self.hidsize

    def set_autograd(self, on: bool = True, state_grad: bool = False, recompute_frames: Optional[int] = None):
        """Opt in to the differentiable forward: in grad mode, with a parameter that requires grad, `forward` returns a latent attached
        to the autograd graph; `state_grad` also attaches the state's K / V, `recompute_frames` re-runs the CNN in the backward instead of
        keeping its activations (see `_PolicyBase.set_autograd`)."""
        recompute_frames = check_recompute_frames(recompute_frames)
        self._autograd = bool(on)
        self._state_grad = bool(on) and bool(state_grad)
        self._recompute_frames = recompute_frames if on else None
        return self

    def initial_state(self, batchsize):
        """lib/policy.py:220-224 -> lib/xf.py:393-397: zeros on the module's device; state_mask None."""
        dev = self.final_ln.weight.device
        mk = lambda: torch.zeros((batchsize, self.cfg.maxlen, self.hidsize), dtype=F32, device=dev)
        return [(None, (mk(), mk())) for _ in range(self.cfg.n_layers)]

    # -- weights -------------------------------------------------------------------------------------------
    def prepared(self) -> _Prepared:
        return self._fold.get()

    def prepared_precise(self):
        return self._fold_fp32.get()

    def prepared_backward(self):
        """The dgrad weights of every layer the trainers' backward runs through (training.py)."""
        return self._bwd.get()

    def _build_prepared(self):
        return _Prepared(self.cfg, dict(self.named_parameters()))

    def _build_prepared_precise(self):
        from .precise import PreparedPrecise
        return PreparedPrecise(self.cfg, dict(self.named_parameters()))

    def _build_backward(self):
        cfg = self.cfg
        P = dict(self.named_parameters())
        w = dict(stacks=[], layers=[])
        pfx = "img_process.cnn"
        for i in range(len(cfg.chans)):
            s = f"{pfx}.stacks.{i}"
            st = dict(convs=[_rot(P[f"{s}.blocks.{j}.conv{k}.layer.weight"]) for j in range(2) for k in range(2)])
            if i > 0 or cfg.first_conv_norm:  # (stack 0's plain first conv has its own backward kernel, ops.firstconv_bwd)
                st["first"] = _rot(P[f"{s}.firstconv.layer.weight"])
            w["stacks"].append(st)
        perm = lambda v: _dense_to_zp(v.detach(), cfg)
        w["dense_t"] = _tr(perm(P[f"{pfx}.dense.layer.weight"]))
        w["dense_g"] = perm(P[f"{pfx}.dense.norm.weight"]).float().contiguous()
        w["dense_b"] = perm(P[f"{pfx}.dense.norm.bias"]).float().contiguous()
        w["linear_t"] = _tr(P["img_process.linear.layer.weight"])
        qkvr = ("q", "k", "v", "r") if cfg.mask_style == "clipped_causal" else ("q", "k", "v")  # R only where the mask has a band
        for l in range(cfg.n_layers):
            o = f"recurrent_layer.blocks.{l}.r.orc_block"
            b = f"recurrent_layer.blocks.{l}"
            cat = torch.cat([P[f"{o}.{c}_layer.weight"] for c in qkvr], 0)
            w["layers"].append(dict(qkvr_t=_tr(cat, cfg.kcat), proj_t=_tr(P[f"{o}.proj_layer.weight"]), mlp0_t=_tr(P[f"{b}.mlp0.layer.weight"]),
                                    mlp1_t=_tr(P[f"{b}.mlp1.layer.weight"])))
        if self.use_lastlayer:
            w["last_t"] = _tr(P["lastlayer.layer.weight"])
        return w

    def _tap(self, name, t):
        if self.debug_taps is not None:
            self.debug_taps[name] = t

    # -- CNN -----------------------------------------------------------------------------------------------
    # Activations are kept in the "ZP" layout [F][H+1][W+1][C] (zero last row / column; include/vpt_b200.h): it lets the
    # conv kernel address every 3x3 neighbour linearly and reuse one shared-memory input span for all nine taps.
    def _cnn_chunk(self, img, prep: _Prepared, out, pfx="img_process.cnn", train=False, stacks=None, record_from=0, plan_frames=None):
        """lib/impala_cnn.py:187-195 for a chunk of frames; writes the last stack's output (ZP [F, Hf+1, Wf+1, C2] bf16) into
        `out` and returns (out, per-frame stats).
        train: the training layout (no stack-norm fold; each residual branch's output `r` kept apart, then `add_zp`), which the
        backward's recompute of a chunk reproduces bit for bit.  stacks: a list that receives, per stack, what the backward needs
        (training layout only; None records nothing), or None for the stacks below `record_from`, which the backward does not enter.
        plan_frames: the convolutions and pools run the launch plan of a chunk of that many frames (None: the chunk's own)."""
        cfg = self.cfg
        conv, pool = ops.conv3x3_zp, ops.maxpool3s2
        if plan_frames is not None:
            conv = functools.partial(ops.conv3x3_zp_plan, plan_frames=plan_frames)
            pool = functools.partial(ops.maxpool3s2_plan, plan_frames=plan_frames)
        H, W = cfg.img_shape[0], cfg.img_shape[1]
        x, mr = None, None
        assert train or stacks is None
        if prep.conv3d is not None:  # IDM: img is (b, T, H, W, 3), whole sequences (the temporal conv needs its neighbours)
            x, mr = ops.conv3d_t5(img, prep.conv3d[0], prep.conv3d[1], cfg.conv3d_out)
            self._tap("conv3d", x)
        for i, c in enumerate(cfg.chans):
            st = prep.stacks[i]
            rec = dict(x_in=x, mr_in=mr, H_in=H, W_in=W, full=None, blocks=[]) if stacks is not None and i >= record_from else None
            fold = self.fold_stack_norm and not train  # inference: the post-pool GroupNorm is folded into its two consumers
            if i == 0 and "fc_w" in st:
                y1, mr1, chan = ops.firstconv_pool(img, st["fc_w"], st["fc_b"], c, zp=True, want_chan=True)
            else:
                Wb, S1, S2 = st["first"]
                full, _ = conv(x, Wb, H, W, mr=mr, S1=S1, S2=S2, relu=1, want_stats=False)
                y1, mr1, chan = pool(full, zp=True, want_chan=True)
                if rec is not None:
                    rec["full"] = full
                del full
            H, W = H // 2, W // 2
            self._tap(f"{pfx}.stacks.{i}.pool", y1)
            if fold and chan is not None:
                # two-norm composition (vpt_norm2_fold): x0 = n(y1) is never written; block 0 reads y1 with per-frame fold tables
                Wb0, tabs = st["conv0n"]
                mrE, Ef, rs, rb = ops.norm2_fold(chan, H * W, st["n_g"], st["n_b"], tabs)
                del chan
                hmid, mrh = conv(y1, Wb0, H, W, mr=mrE, Ef=Ef, relu=1)
                self._tap(f"{pfx}.stacks.{i}.blocks.0.conv0", hmid)
                Wb, S1, S2 = st["convs"][1]
                x, mr = conv(hmid, Wb, H, W, mr=mrh, S1=S1, S2=S2, relu=1, residual=y1, res_scale=rs, res_shift=rb)
                del y1, hmid
                self._tap(f"{pfx}.stacks.{i}.blocks.0", x)
                first_block = 1
            else:
                # post-pool GroupNorm `n` (lib/impala_cnn.py:119) as a pass: the training tape needs x0, and so do shapes whose pool
                # kernel cannot produce per-channel sums
                x, mr = ops.affine_norm_zp(y1, mr1, st["n_g"], st["n_b"])
                if rec is not None:
                    rec.update(y1=y1, mr1=mr1, x0=x, mr0=mr)
                del y1
                self._tap(f"{pfx}.stacks.{i}.n", x)
                first_block = 0
            for j in range(first_block, 2):
                Wb, S1, S2 = st["convs"][2 * j]
                hmid, mrh = conv(x, Wb, H, W, mr=mr, S1=S1, S2=S2, relu=1)
                self._tap(f"{pfx}.stacks.{i}.blocks.{j}.conv0", hmid)
                Wb, S1, S2 = st["convs"][2 * j + 1]
                last = (i == len(cfg.chans) - 1) and j == 1
                if not train:
                    x, mr = conv(hmid, Wb, H, W, mr=mrh, S1=S1, S2=S2, relu=1, residual=x, out=out if last else None)
                else:
                    # training: the branch output r = relu(conv1(..)) is kept on its own (its sign pattern IS the ReLU mask the
                    # backward needs; x + r rounded to bf16 no longer shows which small r were positive), then added
                    r, _ = conv(hmid, Wb, H, W, mr=mrh, S1=S1, S2=S2, relu=1, want_stats=False)
                    x, mr = ops.add_zp(x, r, H, W, out=out if last else None)
                    if rec is not None:
                        rec["blocks"].append(dict(h=hmid, mrh=mrh, r=r, x=x, mr=mr))
                    del r
                self._tap(f"{pfx}.stacks.{i}.blocks.{j}", x)
            if stacks is not None:
                stacks.append(rec)
        return x, mr

    # -- transformer -----------------------------------------------------------------------------------------
    def _linear(self, x, fold, N, *, mr=None, relu=0, residual=None, out=None, out_dtype=None, seg=None, want_stats=False,
                out_scale=1.0, ld_out=None, rowwise=False):
        """rowwise: every row computed as a one-row call computes it (`ops.gemm_rowwise`, the batch-invariant mode)."""
        Wb, S1, S2 = fold
        M, K = x.shape[0], x.shape[1]
        if out is None:
            out = torch.empty((M, N), dtype=out_dtype or BF16, device=x.device)
        part, P = None, ops.gemm_stat_parts(N)
        if want_stats:
            part = torch.empty((M, P, 2), dtype=F32, device=x.device)
        (ops.gemm_rowwise if rowwise else ops.gemm)(x, Wb, out, M, N, K, mr=mr, rows_per_group=1, S1=S1 if mr is not None else None, S2=S2,
                                                    relu=relu, residual=residual, seg=seg, stat_part=part, stat_mode=1 if want_stats else 0,
                                                    out_scale=out_scale, ld_out=ld_out)
        mr_out = ops.stats_finalize(part, M, P, N) if want_stats else None
        return out, mr_out

    def _block(self, l, x, mr_x, first_u8, state, B, t, prep: _Prepared, last: bool, inv: bool = False):
        """lib/util.py:193-211: x_hat = LN(x); y = x_hat + Proj(Attn(x_hat)); z = y + mlp1(relu(mlp0(LN(y)))).
        state: the layer's (mask, (K, V)), or a RingState or RingRows (t = 1), updated in place (returns None for the state).
        inv: the batch-invariant mode (t = 1): row-wise GEMMs and the attention's one-row plan."""
        gemm, attention, attention_ring = ops.gemm, ops.attention, ops.attention_ring
        if inv:
            gemm, attention, attention_ring = ops.gemm_rowwise, ops.attention_plan, ops.attention_ring_plan
        cfg, L = self.cfg, prep.layers[l]
        h, heads, maxlen = cfg.hidsize, cfg.heads, cfg.maxlen
        causal = cfg.mask_style == "clipped_causal"
        ring = state if isinstance(state, _RING_STATES) else None
        xhat, _, _ = ops.affine_norm(x, mr_x, L["ln_g"], L["ln_b"], rows_per_group=1)
        T = maxlen + t
        if ring is not None:  # K / V of the step only (`seg` the identity): ring_write stores them in the ring
            full_k = torch.empty((B, t, h), dtype=BF16, device=x.device)
            full_v = torch.empty((B, t, h), dtype=BF16, device=x.device)
            seg = (t, t, 0)
        else:
            state_mask, (mem_k, mem_v) = state
            full_k = torch.empty((B, T, h), dtype=BF16, device=x.device)
            full_v = torch.empty((B, T, h), dtype=BF16, device=x.device)
            seg = (t, T, maxlen)
        if maxlen > 0 and ring is None:
            if mem_k.shape != (B, maxlen, h):
                raise AssertionError(f"KV memory shape {tuple(mem_k.shape)} != {(B, maxlen, h)}")
            if mem_k.stride() == mem_v.stride() and mem_k.dtype == mem_v.dtype:
                ops.copy_rows2(mem_k, mem_v, 0, full_k, full_v, 0, maxlen)  # lib/xf.py:378-379  full = cat(prev, new), K and V in one launch
            else:
                ops.copy_rows(mem_k, 0, full_k, 0, maxlen)
                ops.copy_rows(mem_v, 0, full_v, 0, maxlen)
        R = None
        if h % 256 == 0:
            # Q | K | V | R as ONE GEMM: K / V land in the rows of `full` after the memory (row remap), R in fp32
            q = torch.empty((B * t, h), dtype=BF16, device=x.device)
            dsts = [(0, q, h, False), (h, full_k, h, True), (2 * h, full_v, h, True)]
            if causal:
                R = torch.empty((B * t, NBASIS * heads), dtype=F32, device=x.device)
                dsts.append((3 * h, R, NBASIS * heads, False))
            Wc, _, bc = L["qkvr"]
            gemm(xhat, Wc, q, B * t, Wc.shape[0], h, S2=bc, seg=seg, dsts=dsts)
        else:  # hidsize not a multiple of the N tile: four launches
            q, _ = self._linear(xhat, L["q"], h, rowwise=inv)
            self._linear(xhat, L["k"], h, out=full_k, seg=seg, ld_out=h, rowwise=inv)
            self._linear(xhat, L["v"], h, out=full_v, seg=seg, ld_out=h, rowwise=inv)
            if causal:
                R, _ = self._linear(xhat, L["r"], NBASIS * heads, out_dtype=F32, rowwise=inv)
        if ring is not None:
            # a view steps some environments: batch row b is ring row idx[b] (-1: an inert row)
            rr, rows = (ring.ring, ring.idx) if isinstance(ring, RingRows) else (ring, None)
            # the step's rows go to their ring slot first: it held memory key 0, which a t = 1 query does not see
            if rr.row_off is None:  # every row at `off`
                ops.ring_write(full_k, full_v, rr.k[l], rr.v[l], rr.mask[l], rr.off, first_u8)
                a = attention_ring(q, rr.k[l], rr.v[l], R, L["b_nd"], first_u8, rr.mask[l], rr.off, heads)
            else:
                ops.ring_write(full_k, full_v, rr.k[l], rr.v[l], rr.mask[l], rr.off, first_u8, rows=rows, row_off=rr.row_off)
                a = attention_ring(q, rr.k[l], rr.v[l], R, L["b_nd"], first_u8, rr.mask[l], rr.off, heads, rows=rows, row_off=rr.row_off)
            new_state = None
        else:
            smask_u8 = state_mask.contiguous().view(torch.uint8) if state_mask is not None else None
            a = attention(q, full_k, full_v, R, L["b_nd"], first_u8, smask_u8, B, t, maxlen, heads, causal=causal)
            # new state (lib/xf.py:380-381: last `maxlen` rows of full; lib/masked_attention.py:86-92)
            new_k = torch.empty((B, maxlen, h), dtype=F32, device=x.device)
            new_v = torch.empty((B, maxlen, h), dtype=F32, device=x.device)
            ops.copy_rows2(full_k, full_v, T - maxlen, new_k, new_v, 0, maxlen)
            new_mask = ops.state_mask_update(smask_u8, first_u8, t, maxlen) if causal else state_mask
            new_state = (new_mask, (new_k, new_v))
        y, mr_y = self._linear(a, L["proj"], h, residual=xhat, want_stats=True, rowwise=inv)
        self._tap(f"recurrent_layer.blocks.{l}.attn", y)
        hmid, _ = self._linear(y, L["mlp0"], h * cfg.pointwise_ratio, mr=mr_y, relu=1, rowwise=inv)
        # the F.relu of lib/policy.py:211 is fused into the last block's epilogue (relu after the residual add)
        z, mr_z = self._linear(hmid, L["mlp1"], h, residual=y, relu=2 if last else 0, want_stats=True, rowwise=inv)
        if not last:
            self._tap(f"recurrent_layer.blocks.{l}", z)
        if self._tape is not None:  # (None for a block below the backward's lowest unit)
            self._tape["blocks"].append(dict(x=x, mr_x=mr_x, xhat=xhat, q=q, full_k=full_k, full_v=full_v, R=R, smask=smask_u8, a=a, y=y,
                                             mr_y=mr_y, hmid=hmid, z=z, mr_z=mr_z) if l >= self._tape["blocks_from"] else None)
        return z, mr_z, new_state

    # -- cached CNN latents -----------------------------------------------------------------------------------
    def _cnn_params(self):
        """The parameters of the CNN part (`CNN_PREFIXES`): the ImpalaCNN with its `dense` layer and, for the IDM, the conv3d pre-stage."""
        return [p for n, p in self.named_parameters() if n.startswith(CNN_PREFIXES)]

    def _cnn_token(self):
        """The token `encode` gives its latents: this network (weakly) and the storage and in-place versions of its CNN parameters, the key
        the kernel-layout copies are rebuilt by (`_Versioned`)."""
        return weakref.ref(self), _fingerprint(self._cnn_params())

    def check_latents(self, lat: FrameLatents):
        """Raises ValueError for latents this network cannot take: not (B, T) of `cnn_outsize` bf16 values with fp32 (mean, rstd), or
        encoded by this very network before its CNN changed (an optimizer step, a load, a move).  Latents of another network with the same
        `cnn_outsize` are accepted: whether its CNN weights are this one's is the caller's responsibility.  No launch."""
        if not isinstance(lat, FrameLatents):
            raise TypeError(f"expected FrameLatents, got {type(lat).__name__}")
        if lat.x.dim() != 3 or lat.x.shape[-1] != self.cfg.cnn_outsize or lat.x.dtype != BF16 or lat.stats.dtype != F32:
            raise ValueError(f"latents must be x bf16 (B, T, {self.cfg.cnn_outsize}) with stats fp32 (B, T, 2) "
                             f"(got x {lat.x.dtype} {tuple(lat.x.shape)}, stats {lat.stats.dtype} {tuple(lat.stats.shape)})")
        if lat.token is not None:
            net, fp = lat.token
            if net() is self and fp != _fingerprint(self._cnn_params()):
                raise ValueError("stale latents: this network's CNN parameters changed (an update, a load or a move) since they were encoded")
        ops.require_cuda(lat.x)

    @torch.no_grad()
    def encode(self, img) -> FrameLatents:
        """The CNN part of the forward (frames -> the `dense` layer's output and its row statistics) in the training layout: the kernels
        and chunks of the trainers' forward with the CNN frozen, so that a step from these latents is bit-identical to that step from the
        frames.  `img` (B, T, H, W, 3), uint8 or float on the uint8 scale as in the forward; bf16 mode only."""
        cfg = self.cfg
        ops.require_cuda(img)
        img = frames_f32(img)
        B, t = img.shape[:2]
        frame_shape = (cfg.img_shape[0], cfg.img_shape[1], 3)
        assert tuple(img.shape[2:]) == frame_shape, f"img shape {tuple(img.shape[2:])} != {frame_shape}"
        if self.precision != "bf16":
            raise NotImplementedError("encode runs in the bf16 mode only (set_precision('bf16'))")
        token = self._cnn_token()
        xd, mr_d = self._cnn_part(img.reshape(B * t, *frame_shape).contiguous(), t, self.prepared(), train=True)
        return FrameLatents(xd.view(B, t, cfg.cnn_outsize), mr_d.view(B, t, 2), token)

    # -- whole net -------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _forward_impl(self, img, first, state_in, invariant: bool = False):
        """img: frames (B, T, H, W, 3), or FrameLatents (B, T): the CNN part is then skipped.  invariant: the batch-invariant mode of a
        one-frame inference call (`MinecraftAgentPolicy.set_batch_invariant`): every launch runs the plan of a one-row call."""
        cfg = self.cfg
        latents = isinstance(img, FrameLatents)
        if latents:
            self.check_latents(img)
        else:
            ops.require_cuda(img)
            img = frames_f32(img)
        B, t = img.shape[:2]
        frame_shape = (cfg.img_shape[0], cfg.img_shape[1], 3)
        if not latents:
            assert tuple(img.shape[2:]) == frame_shape, f"img shape {tuple(img.shape[2:])} != {frame_shape}"
        if isinstance(state_in, _RING_STATES):
            _check_ring_call(self, img, state_in, differentiable=False)
            if isinstance(state_in, RingRows):
                state_in.ring._alloc_row_off()  # (the first step of a view: every row's offset starts at 0)
        else:
            assert len(state_in) == cfg.n_layers, \
                f"Length of state {len(state_in)} did not match length of blocks {cfg.n_layers}"  # lib/util.py:117-119
        if self.precision == "fp32":
            if self._tape is not None:
                raise NotImplementedError("the BC step runs in the bf16 mode only")
            if latents:
                raise NotImplementedError("the forward from latents runs in the bf16 mode only")
            from . import precise
            return precise.forward(self, img, first, state_in)
        if self.precision != "bf16":
            raise ValueError(f"unknown precision {self.precision!r} (use 'bf16' or 'fp32')")
        prep = self.prepared()
        N = B * t
        tape = self._tape
        if latents:
            first_u8 = first.to(device=img.device, dtype=torch.bool).contiguous().view(torch.uint8)
            xd, mr_d = img.x.reshape(N, cfg.cnn_outsize).contiguous(), img.stats.reshape(N, 2).contiguous()
            if tape is not None:  # nothing of the CNN part: the backward stops above the dense layer
                tape.update(prep=prep, xd=xd, mr_d=mr_d, cnn_chunks=[])
        else:
            frames = img.reshape(N, *frame_shape).contiguous()
            first_u8 = first.to(device=img.device, dtype=torch.bool).contiguous().view(torch.uint8)
            xd, mr_d = self._cnn_part(frames, t, prep, train=tape is not None, inv=invariant)
        if tape is not None:
            tape.update(first_u8=first_u8)
        return self._upper_part(xd, mr_d, first_u8, state_in, B, t, prep, inv=invariant)

    def _batch_plan_frames(self, t):
        """Frames per CNN chunk from which every launch plan of this net's CNN is the one of a full chunk (`ops.cnn_batch_plan_frames`);
        the IDM's: whole sequences of t frames."""
        cfg = self.cfg
        H, W = cfg.img_shape[0], cfg.img_shape[1]
        stacks = []
        for c in cfg.chans:
            stacks.append((H, W, c))
            H, W = H // 2, W // 2
        if cfg.conv3d_out is None:
            return ops.cnn_batch_plan_frames(tuple(stacks), self.cnn_chunk_frames)
        n = ops.cnn_batch_plan_frames(tuple(stacks), max(t, self.idm_chunk_frames // t * t))
        return -(-n // t) * t

    def _cnn_part(self, frames, t, prep: _Prepared, train: bool, inv: bool = False):
        """frames [N, H, W, 3] (whole sequences of t frames) -> (xd bf16 [N, cnn_outsize], mr_d fp32 [N, 2]): the conv3d pre-stage (IDM),
        the ImpalaCNN in frame chunks and the dense layer.  train: the training layout (`_cnn_chunk`); with a tape (self._tape) it also
        records what the backward needs.  inv: the batch-invariant mode (inference): every chunk runs the plan of one frame."""
        cfg = self.cfg
        N = frames.shape[0]
        frame_shape = tuple(frames.shape[1:])
        Hf, Wf = cfg.final_hw
        C2 = cfg.chans[-1]
        # ---- ImpalaCNN in frame chunks (bounds the activation workspace), then ONE dense GEMM over all frames
        mrs = []
        tape = self._tape
        # training forward: tape["recompute"] None keeps every stack's activations for the backward (one CNN pass per call); an integer
        # runs the CNN in chunks of that many frames, records nothing per stack, and the backward re-runs each chunk (training.py).
        # Only the stacks from tape["stacks_from"] on are recorded: with the CNN frozen none, and the call may hold several chunks.
        recompute = None if tape is None else tape.get("recompute")
        cnn_bwd = tape is not None and tape["stacks_from"] < len(cfg.chans)
        stacks = tape["stacks"] if cnn_bwd and recompute is None else None
        if cfg.conv3d_out is None:
            step = self.cnn_chunk_frames if recompute is None else min(recompute, self.cnn_chunk_frames)
        else:  # chunks of whole sequences; the IDM's 128-channel full-resolution stage is ~13 MiB/frame
            step = max(1, (self.idm_chunk_frames if recompute is None else min(recompute, self.idm_chunk_frames)) // t) * t
        # Latents promise a frame's output independent of its batch.  The convolutions and pools pick their launch plan by the chunk's
        # frame count, and `dense` by its row count, and a few frames take plans that sum in another order.  So the training layout
        # without a CNN tape (`encode`, a trainer with the CNN frozen) runs a short chunk padded with zero frames (the IDM: zero
        # sequences) up to the count from which every plan is the one of a full chunk, and drops the padded rows after `dense`.
        pad = self._batch_plan_frames(t) if train and not cnn_bwd else 0
        step = max(step, pad)  # (only the last chunk can be short)
        f_last = (N - 1) // step * step
        Nr = f_last + max(N - f_last, pad)  # rows of cnn_out and of the dense GEMM
        cnn_out = torch.empty((Nr, Hf + 1, Wf + 1, C2), dtype=BF16, device=frames.device)
        for f0 in range(0, N, step):
            F_ = min(step, N - f0)
            Fr = min(step, Nr - f0)
            chunk = frames[f0:f0 + F_]
            if Fr > F_:
                chunk = torch.cat([chunk, chunk.new_zeros((Fr - F_, *frame_shape))])
            if cfg.conv3d_out is not None:
                chunk = chunk.view(Fr // t, t, *frame_shape)
            _, mr = self._cnn_chunk(chunk, prep, cnn_out[f0:f0 + Fr], train=train, stacks=stacks,
                                    record_from=0 if tape is None else tape["stacks_from"], plan_frames=1 if inv else None)
            mrs.append(mr)
        mr_c = mrs[0] if len(mrs) == 1 else torch.cat(mrs, 0)
        Kd = (Hf + 1) * (Wf + 1) * C2  # ZP rows flattened; the zero row / column meets zero weight columns
        xd, mr_d = self._linear(cnn_out.view(Nr, Kd), prep.dense, cfg.cnn_outsize, mr=mr_c, relu=1, want_stats=True, rowwise=inv)
        if Nr > N:
            cnn_out, mr_c, xd, mr_d = cnn_out[:N], mr_c[:N], xd[:N], mr_d[:N]
        if tape is not None:
            assert not (cnn_bwd and recompute is None and len(mrs) != 1), "the stored tape holds one CNN chunk (training._Trainer.check_call)"
            tape.update(prep=prep, frames=frames, cnn_out=cnn_out, mr_c=mr_c, xd=xd, mr_d=mr_d,
                        cnn_chunks=[(f0, min(f0 + step, N)) for f0 in range(0, N, step)] if cnn_bwd else [])
        return xd, mr_d

    def _upper_part(self, xd, mr_d, first_u8, state_in, B, t, prep: _Prepared, inv: bool = False):
        """(xd, mr_d) of `_cnn_part` or of cached latents -> img_process.linear -> the transformer -> lastlayer -> final_ln:
        (latent bf16 [N, h], latent fp32 (B, t, h), state_out).  Records into the tape (self._tape) when there is one."""
        cfg = self.cfg
        tape = self._tape
        self._tap("img_process.cnn.dense", xd)
        x, mr_x = self._linear(xd, prep.linear, cfg.hidsize, mr=mr_d, relu=1, want_stats=True, rowwise=inv)
        self._tap("img_process", x)
        if tape is not None:
            tape.update(x0=x, mr_x0=mr_x)
        # ---- transformer
        ring = isinstance(state_in, _RING_STATES)
        state_out = state_in if ring else []
        for l in range(cfg.n_layers):
            x, mr_x, s = self._block(l, x, mr_x, first_u8, state_in if ring else state_in[l], B, t, prep, last=(l == cfg.n_layers - 1), inv=inv)
            if not ring:
                state_out.append(s)
        # every layer has written its row at its slot: the next step's oldest row is one further on
        if isinstance(state_in, RingRows):
            ops.ring_advance_rows(state_in.ring.row_off, state_in.idx, cfg.maxlen)
        elif ring:
            ops.ring_advance(state_in.off, cfg.maxlen)
        # x is relu(recurrent output) here
        if self.use_lastlayer:
            z_last, mr_zl = x, mr_x
            x, mr_x = self._linear(x, prep.last, cfg.hidsize, mr=mr_x, relu=1, want_stats=True, rowwise=inv)
            if tape is not None:
                tape.update(z_last=z_last, mr_zl=mr_zl, xl=x, mr_xl=mr_x)
        lat_bf16, lat_f32, _ = ops.affine_norm(x, mr_x, prep.fin_g, prep.fin_b, rows_per_group=1, want_f32=True)
        return lat_bf16, lat_f32.view(B, t, cfg.hidsize), state_out

    def forward(self, ob, state_in, context):
        """lib/policy.py:193-218."""
        first = context["first"]
        img = _ob_input(ob)
        if isinstance(state_in, _RING_STATES):
            _check_ring_call(self, img, state_in, _differentiable(self, img))
        if _differentiable(self, img):
            (latent,), state_out = _autograd_runner(self).run(img, first, state_in)
        else:
            _, latent, state_out = self._forward_impl(img, first, state_in)
        if self.single_output:
            return latent, state_out
        return (latent, latent), state_out


class InverseActionNet(MinecraftPolicy):
    """lib/policy.py:342-403: conv3d pre-stage -> ImpalaCNN (first conv normalised) -> unmasked transformer ->
    relu -> final_ln.  `lastlayer` keeps its parameters (state_dict schema) but its output is discarded by the reference
    (lib/policy.py:390-391), so it is not computed."""

    use_lastlayer = False

    def __init__(self, hidsize=512, conv3d_params=None, **MCPoliy_kwargs):
        super().__init__(hidsize=hidsize, conv3d_params=conv3d_params, **MCPoliy_kwargs)

    def forward(self, ob, state_in, context):
        """lib/policy.py:374-392 -> ((pi_latent, None), state_out)."""
        first = context["first"]
        img = _ob_input(ob)
        if isinstance(state_in, _RING_STATES):
            _check_ring_call(self, img, state_in, _differentiable(self, img))
        if _differentiable(self, img):
            (latent,), state_out = _autograd_runner(self).run(img, first, state_in)
        else:
            _, latent, state_out = self._forward_impl(img, first, state_in)
        return (latent, None), state_out


# ---------------------------------------------------------------------------------------------------------------
# heads + MinecraftAgentPolicy
# ---------------------------------------------------------------------------------------------------------------
class _PolicyBase(nn.Module):
    """Shared head plumbing of MinecraftAgentPolicy and InverseActionPolicy (lib/action_head.py:136-260)."""

    has_value_head = True
    graph_relayout = True  # `refresh_weights` as one CUDA graph replay (False: the copies are rebuilt eagerly on use)

    def _init_heads(self, action_space, pi_head_kwargs):
        self.action_space = action_space
        self.temperature = float((pi_head_kwargs or {}).get("temperature", 1.0))
        h = self.net.output_latent_size()
        if self.has_value_head:  # lib/scaled_mse_head.py:24 + lib/normalize_ewma.py:18-20
            w, b = _default_linear(1, h)
            _set(self, "value_head.linear.weight", w)
            _set(self, "value_head.linear.bias", b)
            _set(self, "value_head.normalizer.running_mean", torch.zeros(1), requires_grad=False)
            _set(self, "value_head.normalizer.running_mean_sq", torch.zeros(1), requires_grad=False)
            _set(self, "value_head.normalizer.debiasing_term", torch.tensor(0.0), requires_grad=False)
        # pi head: lib/action_head.py:263-275 -> one CategoricalActionHead per Discrete TensorType, in dict order
        self.head_specs = OrderedDict()
        self.pi_head = _DictActionHead()
        for name, space in action_space.items():
            n = space.eltype.n
            shape = tuple(space.shape)
            cnt = 1
            for s_ in shape:
                cnt *= s_
            self.pi_head.add_module(name, _CategoricalActionHead(shape, n))
            w, b = _default_linear(cnt * n, h)
            _set(self, f"pi_head.{name}.linear_layer.weight", w)
            _set(self, f"pi_head.{name}.linear_layer.bias", b)
            self.head_specs[name] = (shape, n)
        self._heads_fold = _Versioned(self._head_params, self._build_heads_prepared)
        self._heads_fold_fp32 = _Versioned(self._head_params, self._build_heads_prepared_precise)
        self._heads_bwd = {}       # tuple of head layers -> _Versioned heads_t (`_heads_prepared_backward`)
        self._relayout = None      # (parameter pointers, copies, CUDA graph, graph-owned layouts) of `refresh_weights`
        self._relayout_seen = 0
        self._autograd = False  # set_autograd
        self._state_grad = False
        self._recompute_frames = None
        self._ag_runner = None

    def initial_state(self, batch_size: int):
        return self.net.initial_state(batch_size)

    def set_autograd(self, on: bool = True, state_grad: bool = False, recompute_frames: Optional[int] = None):
        """Opt in to the differentiable forward (also for `self.net` called on its own).  When on, a forward in grad mode (not inference
        mode) with at least one parameter that requires grad runs the training forward (no stack-norm fold; within the 1e-2 tolerance of
        the inference path, not bit-identical to it) as an autograd `Function` whose backward is the trainers' hand-written one, so that
        `loss.backward()` accumulates into `.grad`.  pd and vpred are attached to the graph; `state_out` is detached and a `state_in`
        that requires grad raises (no gradient through the KV memory, behavioural_cloning.py:109-111).  With recompute_frames=None at
        most `net.cnn_chunk_frames` (2048) frames per call (the IDM: `net.idm_chunk_frames` (512)); always T <= 128 for the IDM and bf16
        mode only.  A parameter that only feeds outputs the loss does not use gets None, as in the reference.  `act`, `predict`, `v` and
        `GraphedAct` stay inference-only.

        state_grad=True (truncated backpropagation through time across calls): `state_out`'s K / V are attached to the graph too and a
        `state_in` whose K / V require grad is accepted, so a loss on a later call trains this one through the KV memory.  Truncate with
        `state = tree_map(detach)` every k calls and call `backward()` once per window: every call of the window keeps its tape (its
        activations) until then.  Each call keeps its own limits.  No effect on a model without memory (the IDM).

        recompute_frames=F (a positive int): the forward runs the ImpalaCNN in chunks of F frames (at most `net.cnn_chunk_frames`; the
        IDM rounds F down to whole sequences, at least one) and keeps only its output, and the backward re-runs each chunk's forward
        before back-propagating through it.  That costs one more CNN forward per call and frees the CNN activations, nearly all of a
        call's tape (20.7 MiB per frame at 2x width with its backward workspace, measured on an H100: README), so a call or a BPTT window can hold many more frames:
        up to `training._Trainer.max_call_frames` per call.  The gradients are those of the stored tape (bit-identical when one chunk
        holds the call).  None keeps the activations (faster when they fit).

        Frozen parameters (requires_grad=False when the forward runs) get no gradient and the backward skips the work that only served
        them, stopping at the lowest unit that trains; with the ImpalaCNN frozen the forward keeps none of its activations and the
        stored-tape frame limit does not apply.

        An `img` that requires grad (a floating dtype on the uint8 scale, `frames_f32`) makes the forward differentiable even with every
        parameter frozen, and `loss.backward()` then writes `img.grad`; the trainable parameters' gradients are those of the same call
        without it, bit for bit.

        The forward also takes cached latents, `{"img_latent": policy.encode(img)}`, with every parameter of the CNN part (`img_process.cnn.*`,
        the IDM's `conv3d_layer.*`) frozen (ValueError otherwise, before any launch): no CNN runs, forward or backward, the gradients are those
        of the same call from `img` with the CNN frozen, and the limits are `max_call_frames` / `max_call_batch`, T <= 128 for the IDM and
        the bf16 mode; `recompute_frames` has nothing to recompute and is ignored for such a call.  Latents carry no graph (no image
        gradient)."""
        recompute_frames = check_recompute_frames(recompute_frames)
        self._autograd = bool(on)
        self._state_grad = bool(on) and bool(state_grad)
        self._recompute_frames = recompute_frames if on else None
        self.net.set_autograd(on, state_grad=state_grad, recompute_frames=recompute_frames)
        return self

    def encode(self, img) -> FrameLatents:
        """`self.net.encode(img)`: the CNN part of the forward, once, for frames whose CNN output is used again (the epochs of a BC
        fine-tune, the PPO epochs over one rollout, the frozen reference policy): `policy({"img_latent": lat}, first, state)` and the
        trainers' `loss_and_grad(lat, ...)` then run the rest.  See `MinecraftPolicy.encode` and INTEGRATION.md, "cached latents"."""
        return self.net.encode(img)

    def set_precision(self, precision: str):
        """"bf16" (default, production: bf16 operands, 1e-2 tolerance) or "fp32" (fp32-parity mode, precise.py: 1e-3 tolerance)."""
        if precision not in ("bf16", "fp32"):
            raise ValueError("precision must be 'bf16' or 'fp32'")
        self.net.precision = precision
        return self

    # -- kernel-layout copies of the head weights, and their re-layout after an optimizer step ------------------
    def _head_params(self):
        """The parameters of the heads' kernel-layout copies.  The EWMA normaliser is in none of them: an RL step updates it on every call,
        and `denormalize` caches its own scalars."""
        return [*self.pi_head.parameters(), *(self.value_head.linear.parameters() if self.has_value_head else ())]

    def _heads_prepared(self):
        return self._heads_fold.get()

    def _heads_prepared_precise(self):
        return self._heads_fold_fp32.get()

    def _heads_prepared_backward(self, layers):
        """heads_t, the dgrad weight bf16 [h][ld] of the given head layers (the column blocks of the trainers' logits gradient, in order),
        zero-padded to a multiple of 8 columns.  One copy per list of layers: the BC and IDM steps use the action heads, the RL step and
        the differentiable forward the value head as well."""
        key = tuple(layers)
        if key not in self._heads_bwd:
            self._heads_bwd[key] = _Versioned(self._head_params, functools.partial(self._build_heads_backward, key))
        return self._heads_bwd[key].get()

    def _pi_matrix(self):
        """The action heads as one linear layer: (weight [ntot][h], bias [ntot], {name: (first column, width)}, ntot)."""
        ws, bs, cols, c0 = [], [], OrderedDict(), 0
        for name in self.head_specs:
            lin = getattr(self.pi_head, name).linear_layer
            ws.append(lin.weight.detach())
            bs.append(lin.bias.detach())
            cols[name] = (c0, lin.weight.shape[0])
            c0 += lin.weight.shape[0]
        return torch.cat(ws, 0), torch.cat(bs, 0), cols, c0

    def _build_heads_prepared(self):
        W, b, cols, ntot = self._pi_matrix()
        hp = dict(pi=_fold_linear(W, bias=b), cols=cols, ntot=ntot)
        if self.has_value_head:
            hp["v"] = _fold_linear(self.value_head.linear.weight.detach(), bias=self.value_head.linear.bias.detach())
        return hp

    def _build_heads_prepared_precise(self):
        from .precise import _f, _split_w
        W, b, cols, ntot = self._pi_matrix()
        hp = dict(pi=(_split_w(W), _f(b)), cols=cols, ntot=ntot)
        if self.has_value_head:
            hp["v"] = (_split_w(self.value_head.linear.weight), _f(self.value_head.linear.bias))
        return hp

    def _build_heads_backward(self, layers):
        rows = sum(lin.weight.shape[0] for lin in layers)
        return _tr(torch.cat([lin.weight for lin in layers], 0), (rows + 7) // 8 * 8)

    def refresh_weights(self):
        """Re-layout after an optimizer step of the copies training uses (net forward folds and backward transposes, head folds, every
        `heads_t` asked for); called by the trainers and the differentiable forward, a no-op when nothing changed.  Eagerly ~500 small
        launches; the parameters live at fixed addresses (FlatAdamDP's bucket), so from the second refresh on it is ONE captured CUDA
        graph replay writing the same tensors in place.  No parameter changes between a forward and its backward (the trainers run both
        in one call, the differentiable forward's version check refuses it), so no tape's layouts are rewritten before its backward."""
        caches = [self.net._fold, self._heads_fold, self.net._bwd, *self._heads_bwd.values()]
        if not any(c.stale() for c in caches):
            return
        if not self.graph_relayout or not all(p.is_cuda for p in self.parameters()):
            return  # the getters rebuild eagerly on use
        ptrs = tuple(p.data_ptr() for p in self.parameters())
        if self._relayout is not None and (self._relayout[0] != ptrs or self._relayout[1] != caches):
            self._relayout = None  # the parameters moved (e.g. .to(), a new optimizer bucket) or a new heads_t was asked for: capture again
        if self._relayout is None:
            self._relayout_seen += 1
            if self._relayout_seen < 2:
                return  # first change: eager (also warms up every lazily initialised helper before capture)
            g = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            with torch.no_grad(), torch.cuda.graph(g):
                values = [c.build() for c in caches]
            self._relayout = (ptrs, caches, g, values)
        _, caches, g, values = self._relayout
        g.replay()
        for c, v in zip(caches, values):
            c.set(v)

    def __getstate__(self):
        return {**super().__getstate__(), "_relayout": None, "_relayout_seen": 0}  # a copy captures its own graph (a CUDA graph cannot be copied)

    @torch.no_grad()
    def _heads(self, lat_bf16, B, t, mask=None, rowwise=False):
        """lib/action_head.py:163-174 for every head + lib/scaled_mse_head.py:34-35.  rowwise: the batch-invariant mode's GEMMs."""
        if isinstance(lat_bf16, tuple):  # fp32-parity mode: (latent hi, latent lo)
            from . import precise
            return precise.heads(self, lat_bf16, B, t, mask)
        hp = self._heads_prepared()
        N = lat_bf16.shape[0]
        ntot = hp["ntot"]
        ld = (ntot + 7) // 8 * 8
        raw = torch.empty((N, ld), dtype=F32, device=lat_bf16.device)
        self.net._linear(lat_bf16, hp["pi"], ntot, out=raw, out_scale=1.0 / self.temperature, ld_out=ld, rowwise=rowwise)
        pd = OrderedDict()
        for name, (shape, n) in self.head_specs.items():
            c0, width = hp["cols"][name]
            cnt = width // n
            if mask is not None and mask.get(name) is not None:
                # lib/action_head.py:170-171: shaped_out[~mask] = LOG0 (-100) before the log-softmax.  Rare side input:
                # applied as a masked fill on the raw (already temperature-scaled) logits.
                view = raw[:, c0:c0 + width].view(B, t, *shape, n)
                view.masked_fill_(~mask[name].to(device=raw.device, dtype=torch.bool).expand_as(view), -100.0)
            if cnt == 1:
                lp = ops.log_softmax(raw, c0, n)
            else:  # several sub-actions per head (IDM): softmax over each group of n columns
                lp = torch.cat([ops.log_softmax(raw, c0 + i * n, n) for i in range(cnt)], dim=1)
            pd[name] = lp.view(B, t, *shape, n)
        if not self.has_value_head:
            return pd, None
        vpred, _ = self.net._linear(lat_bf16, hp["v"], 1, out_dtype=F32, rowwise=rowwise)
        return pd, vpred.view(B, t, 1)
    # -- distribution helpers (lib/action_head.py:176-220, 250-260): the reference's policy calls them on its pi_head --------------
    def sample(self, pd, deterministic: bool = False):
        """`pi_head.sample`."""
        return self.pi_head.sample(pd, deterministic)

    def logprob(self, ac, pd):
        """`pi_head.logprob`."""
        return self.pi_head.logprob(ac, pd)


class _CategoricalActionHead(_Node):
    """lib/action_head.py:136-220 on the kernels: the distribution methods of one categorical head, whose log-probs `pd` have the shape
    (..., *shape, n).  Holds the head's `linear_layer` parameters (the policy's forward computes every head's logits in one GEMM, `_heads`).
    `entropy` and `kl_divergence` are differentiable (autograd `Function`s on their backward kernels) in any input that requires grad."""

    def __init__(self, shape, num_actions: int):
        super().__init__()
        self.num_actions = num_actions
        self.output_shape = tuple(shape) + (num_actions,)

    def _rows(self, logits):
        """-> (the leading shape, fp32 [rows, groups*n] with unit column stride, groups)."""
        k = len(self.output_shape)
        if tuple(logits.shape[logits.dim() - k:]) != self.output_shape:
            raise ValueError(f"log-probs of shape {tuple(logits.shape)} do not end in the head's {self.output_shape}")
        groups = math.prod(self.output_shape[:-1])
        x = logits.reshape(-1, groups * self.num_actions).to(F32)
        return logits.shape[:logits.dim() - k], (x if x.stride(1) == 1 else x.contiguous()), groups

    def logprob(self, actions, logits):
        """log p(actions) summed over the head's sub-actions: shape (...)."""
        lg = logits.contiguous()
        idx = actions.to(torch.int64)
        if lg.requires_grad and torch.is_grad_enabled():
            lp = _GatherLogprob.apply(lg, idx)  # pd from the differentiable forward
        else:
            lp = ops.gather_logprob(lg, idx)
        for _ in self.output_shape[:-1]:
            lp = lp.sum(dim=-1)
        return lp

    def sample(self, logits, deterministic: bool = False, keys=None, seed: int = 0, head: int = 0):
        """Gumbel-max sample (or the argmax); `torch.rand_like` supplies the uniforms so the Philox stream is consumed exactly like the
        reference's (lib/action_head.py:200).  keys: device int64 (rows, 2) of (stream, step), one per row of the head's logits: the
        counter-based noise of `ops.gumbel_argmax_keyed` under `seed`, with `head` the head's index (the batch-invariant mode)."""
        lg = logits.contiguous()
        if keys is not None and not deterministic:
            return ops.gumbel_argmax_keyed(lg, keys, seed, head)
        u = None if deterministic else torch.rand_like(lg)
        return ops.gumbel_argmax(lg, u)

    def entropy(self, logits):
        """-sum exp(logits) * logits over the classes and the sub-actions: shape (...)."""
        lead, x, groups = self._rows(logits)
        if x.requires_grad and torch.is_grad_enabled():
            ent = _HeadEntropy.apply(x, groups)
        else:
            ent = ops.head_entropy(x, groups)
        return ent.view(lead)

    def kl_divergence(self, logits_q, logits_p):
        """KL(q || p) = sum exp(logits_q) * (logits_q - logits_p) over the classes and the sub-actions: shape (..., 1), the reference's
        `keepdim` (lib/action_head.py:216-220)."""
        lead, q, groups = self._rows(logits_q)
        lead_p, p, _ = self._rows(logits_p)
        if lead_p != lead:
            raise ValueError(f"kl_divergence: log-probs of shapes {tuple(logits_q.shape)} and {tuple(logits_p.shape)}")
        if (q.requires_grad or p.requires_grad) and torch.is_grad_enabled():
            kl = _HeadKL.apply(q, p, groups)
        else:
            kl = ops.head_kl(q, p, groups)
        return kl.view(*lead, 1)


class _DictActionHead(_Node):
    """lib/action_head.py:223-260: the policy's `pi_head`, one `_CategoricalActionHead` per action, in the action space's order.  Each
    method takes dicts of per-head tensors and sums the heads' results (a dict of samples for `sample`)."""

    def __getitem__(self, key):
        return self._modules[key]

    def __iter__(self):
        return iter(self._modules)

    def __len__(self):
        return len(self._modules)

    def keys(self):
        return self._modules.keys()

    def values(self):
        return self._modules.values()

    def items(self):
        return self._modules.items()

    @staticmethod
    def _sum(parts):
        tot = None
        for x in parts:
            tot = x if tot is None else tot + x
        return tot

    def logprob(self, actions, logits):
        return self._sum(head.logprob(actions[k], logits[k]) for k, head in self.items())

    def sample(self, logits, deterministic: bool = False, keys=None, seed: int = 0):
        """keys, seed: `_CategoricalActionHead.sample`; head i (in this dict's order) draws with head index i."""
        if keys is None:
            return OrderedDict((k, head.sample(logits[k], deterministic)) for k, head in self.items())
        return OrderedDict((k, head.sample(logits[k], deterministic, keys=keys, seed=seed, head=i)) for i, (k, head) in enumerate(self.items()))

    def entropy(self, logits):
        return self._sum(head.entropy(logits[k]) for k, head in self.items())

    def kl_divergence(self, logits_q, logits_p):
        return self._sum(head.kl_divergence(logits_q[k], logits_p[k]) for k, head in self.items())


def _no_double_backward():
    if torch.is_grad_enabled():
        raise NotImplementedError("the head distribution kernels have no double backward (create_graph=True)")


class _HeadEntropy(torch.autograd.Function):
    """`ops.head_entropy` attached to the graph; the backward is `ops.head_entropy_bwd`."""

    @staticmethod
    def forward(ctx, lp, groups):
        ctx.save_for_backward(lp)
        ctx.groups = groups
        return ops.head_entropy(lp, groups)

    @staticmethod
    def backward(ctx, g):
        _no_double_backward()
        (lp,) = ctx.saved_tensors
        return ops.head_entropy_bwd(lp, g.to(F32).contiguous(), ctx.groups), None


class _HeadKL(torch.autograd.Function):
    """`ops.head_kl` attached to the graph; the backward (`ops.head_kl_bwd`) computes only the sides that require grad."""

    @staticmethod
    def forward(ctx, lq, lp, groups):
        ctx.save_for_backward(lq, lp)
        ctx.groups = groups
        return ops.head_kl(lq, lp, groups)

    @staticmethod
    def backward(ctx, g):
        _no_double_backward()
        lq, lp = ctx.saved_tensors
        dq, dp = ops.head_kl_bwd(lq, lp, g.to(F32).contiguous(), ctx.groups, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return dq, dp, None


class _GatherLogprob(torch.autograd.Function):
    """`ops.gather_logprob` on log-probs attached to the graph: the same values; the backward scatters the gradient to the chosen class."""

    @staticmethod
    def forward(ctx, logits, idx):
        ctx.save_for_backward(idx)
        ctx.shape = logits.shape
        return ops.gather_logprob(logits, idx)

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        d = torch.zeros(ctx.shape, dtype=F32, device=g.device)
        d.scatter_(-1, idx.reshape(*ctx.shape[:-1], 1), g.reshape(*ctx.shape[:-1], 1).to(F32))
        return d, None


class MinecraftAgentPolicy(_PolicyBase):
    """lib/policy.py:227-339."""

    def __init__(self, action_space, policy_kwargs, pi_head_kwargs):
        super().__init__()
        self.net = MinecraftPolicy(**policy_kwargs)
        self._init_heads(action_space, pi_head_kwargs)
        self._denorm = _Versioned(self.value_head.normalizer.parameters, self._build_denorm)
        self.batch_invariant, self.noise_seed = False, 0

    def set_batch_invariant(self, on: bool = True, seed: int = 0):
        """The batch-invariant mode of one-frame inference steps (`act`, `v`, `get_output_for_observation`, `forward` with T = 1; frames or
        latents; a pytree state, a RingState or a view; eager or through `GraphedAct`).  Every output of a row (pd, vpred, log_prob, the
        K / V row and mask it stores) then equals, bit for bit, the default-mode B = 1 step of that environment alone, whatever the batch,
        the row's position, the other rows and the padding: every launch runs the plan of a one-row call.  A sampled action comes from
        counter-based noise keyed by (seed, stream, step, head, column) (`ops.gumbel_argmax_keyed`): a ring's step of environment e uses
        (e, RingState.steps[e]), a pytree `act` the caller's `noise_keys`.  Read when a call runs.  The differentiable forward and the
        trainers ignore it.  Returns the policy."""
        self.batch_invariant, self.noise_seed = bool(on), int(seed)
        return self

    def _invariant_call(self, t, differentiable: bool):
        """Whether a forward call runs in the batch-invariant mode; raises, before any launch, for one the mode cannot serve."""
        if not self.batch_invariant or differentiable:
            return False
        if self.net.precision != "bf16":
            raise NotImplementedError("the batch-invariant mode runs in the bf16 mode only (set_precision('bf16'))")
        if t != 1:
            raise ValueError(f"the batch-invariant mode is for one-frame steps (T = 1, got T = {t})")
        return True

    def _check_noise_keys(self, B, state_in, sample: bool, noise_keys):
        """Raises, before any launch, for `noise_keys` an `act` call cannot take or a keyed sample without them."""
        if noise_keys is not None:
            if not self.batch_invariant:
                raise ValueError("noise_keys are for the batch-invariant mode (set_batch_invariant)")
            if isinstance(state_in, _RING_STATES):
                raise ValueError("a ring step samples with the keys of RingState.steps: noise_keys are for a pytree state")
            if (not torch.is_tensor(noise_keys) or noise_keys.dtype != torch.int64 or tuple(noise_keys.shape) != (B, 2)
                    or not noise_keys.is_contiguous()):
                raise ValueError(f"noise_keys must be a contiguous CUDA int64 ({B}, 2) of (stream, step) (got "
                                 f"{getattr(noise_keys, 'dtype', type(noise_keys))} {tuple(getattr(noise_keys, 'shape', ()))})")
            ops.require_cuda(noise_keys)
        elif self.batch_invariant and sample and not isinstance(state_in, _RING_STATES):
            raise ValueError("a stochastic act on a pytree state in the batch-invariant mode needs noise_keys, (B, 2) of (stream, step): "
                             "keys from the row's position would make its action depend on the batch")

    def forward(self, obs, first: torch.Tensor, state_in):
        """lib/policy.py:252-269 -> ((pi_logits, vpred, None), state_out)."""
        if isinstance(obs, dict):
            obs = obs.copy()
            mask = obs.pop("mask", None)
        else:
            mask = None
        img = _ob_input(obs)
        if isinstance(state_in, _RING_STATES):
            _check_ring_call(self.net, img, state_in, _differentiable(self, img))
        inv = self._invariant_call(img.shape[1], _differentiable(self, img))
        if _differentiable(self, img):
            outs, state_out = _autograd_runner(self).run(img, first, state_in, mask)
            pi_logits = OrderedDict(zip(self.head_specs, outs[:-1]))
            return (pi_logits, outs[-1], None), state_out
        lat_bf16, _, state_out = self.net._forward_impl(img, first, state_in, invariant=inv)
        B, t = img.shape[:2]
        pi_logits, vpred = self._heads(lat_bf16, B, t, mask, rowwise=inv)
        return (pi_logits, vpred, None), state_out

    def denormalize(self, v):
        """lib/normalize_ewma.py:31-35,57-60 (a 3-scalar affine map; host-side glue)."""
        std, mean = self._denorm.get()  # the scalars only change when the normaliser is updated / reloaded:
        return v * std + mean           # 7 of the 9 tiny launches per rollout step were their recomputation

    def _build_denorm(self):
        nz = self.value_head.normalizer
        deb = nz.debiasing_term.clamp(min=1e-5)
        mean = nz.running_mean / deb
        var = (nz.running_mean_sq / deb - mean ** 2).clamp(min=1e-2)
        return torch.sqrt(var)[None, None], mean[None, None]

    def get_logprob_of_action(self, pd, action):
        """lib/policy.py:271-279."""
        ac = {k: v.unsqueeze(1) for k, v in action.items()}
        log_prob = self.logprob(ac, pd)
        assert not torch.isnan(log_prob).any()
        return log_prob[:, 0]

    def get_kl_of_action_dists(self, pd1, pd2):
        """lib/policy.py:281-285: KL(pd1 || pd2) per frame, shape (..., 1)."""
        return self.pi_head.kl_divergence(pd1, pd2)

    def get_output_for_observation(self, obs, state_in, first):
        """lib/policy.py:287-305.  obs["img"] (B, H, W, 3) or obs["img_latent"], FrameLatents (B,)."""
        obs = {k: _add_time(v) for k, v in obs.items()}
        first = first.unsqueeze(1)
        (pd, vpred, _), state_out = self(obs=obs, first=first, state_in=state_in)
        return pd, self.denormalize(vpred)[:, 0], state_out

    @torch.no_grad()
    def act(self, obs, first, state_in, stochastic: bool = True, taken_action=None, return_pd=False, noise_keys=None):
        """lib/policy.py:307-328.  noise_keys: the batch-invariant mode's sampling keys for a pytree state, a CUDA int64 (B, 2) of
        (stream, step) per row (`set_batch_invariant`; a ring step takes (e, RingState.steps[e]) and advances `steps`)."""
        self._check_noise_keys(first.shape[0], state_in, stochastic and taken_action is None, noise_keys)
        obs = {k: v.unsqueeze(1) for k, v in obs.items()}
        first = first.unsqueeze(1)
        (pd, vpred, _), state_out = self(obs=obs, first=first, state_in=state_in)
        keys = noise_keys
        if self.batch_invariant and isinstance(state_in, _RING_STATES):
            ring, rows = (state_in.ring, state_in.idx) if isinstance(state_in, RingRows) else (state_in, None)
            keys = ops.ring_noise_keys(ring._alloc_steps(), rows, ring.batch_size)
        if taken_action is None and keys is not None:
            ac = self.pi_head.sample(pd, deterministic=not stochastic, keys=keys, seed=self.noise_seed)
        elif taken_action is None:
            ac = self.sample(pd, deterministic=not stochastic)
        else:
            ac = {k: v.unsqueeze(1) for k, v in taken_action.items()}
        log_prob = self.logprob(ac, pd)
        if not (log_prob.is_cuda and torch.cuda.is_current_stream_capturing()):  # the check synchronises: not inside a graph capture
            assert not torch.isnan(log_prob).any()
        result = {"log_prob": log_prob[:, 0], "vpred": self.denormalize(vpred)[:, 0]}
        if return_pd:
            result["pd"] = {k: v[:, 0] for k, v in pd.items()}
        ac = {k: v[:, 0] for k, v in ac.items()}
        return ac, state_out, result

    def make_graphed_act(self, batch_size: int, pdl: bool = False, memory: str = "pytree", envs: Optional[int] = None):
        """Rollout-latency path (agent.py:190-206, SURVEY f-1): returns a callable with the signature of `act` whose whole
        step (forward + heads + sampling + log-prob + KV-memory roll) is ONE captured CUDA graph replay (pdl: captured with
        programmatic dependent launch between its kernels -- bit-identical; memory, envs: see `GraphedAct`)."""
        return GraphedAct(self, batch_size, pdl=pdl, memory=memory, envs=envs)

    @torch.no_grad()
    def v(self, obs, first, state_in):
        """lib/policy.py:330-339."""
        obs = {k: v.unsqueeze(1) for k, v in obs.items()}
        first = first.unsqueeze(1)
        (pd, vpred, _), state_out = self(obs=obs, first=first, state_in=state_in)
        return self.denormalize(vpred)[:, 0]


class InverseActionPolicy(_PolicyBase):
    """lib/policy.py:406-467 (the IDM): InverseActionNet + factored categorical heads, no value head."""

    has_value_head = False

    def __init__(self, action_space, pi_head_kwargs=None, idm_net_kwargs=None):
        super().__init__()
        self.net = InverseActionNet(**idm_net_kwargs)
        self._init_heads(action_space, pi_head_kwargs)

    def forward(self, obs, first: torch.Tensor, state_in, **kwargs):
        """lib/policy.py:432-446 -> ((pi_logits, None, None), state_out)."""
        if isinstance(obs, dict):
            obs = obs.copy()
            mask = obs.pop("mask", None)
        else:
            mask = None
        img = _ob_input(obs)
        if isinstance(state_in, _RING_STATES):
            _check_ring_call(self.net, img, state_in, _differentiable(self, img))
        if _differentiable(self, img):
            outs, state_out = _autograd_runner(self).run(img, first, state_in, mask)
            return (OrderedDict(zip(self.head_specs, outs)), None, None), state_out
        lat_bf16, _, state_out = self.net._forward_impl(img, first, state_in)
        B, t = img.shape[:2]
        pi_logits, _ = self._heads(lat_bf16, B, t, mask)
        return (pi_logits, None, None), state_out

    @torch.no_grad()
    def predict(self, obs, deterministic: bool = True, **kwargs):
        """lib/policy.py:448-464."""
        (pd, _, _), state_out = self(obs=obs, **kwargs)
        ac = self.sample(pd, deterministic=deterministic)
        log_prob = self.logprob(ac, pd)
        assert not torch.isnan(log_prob).any()
        return ac, state_out, {"log_prob": log_prob, "pd": pd}


class GraphedAct:
    """`MinecraftAgentPolicy.act` for a fixed batch size as a CUDA graph: ~170 kernel launches become one graph launch,
    which is what bounds the B=1, T=1 rollout step (the arithmetic itself is ~0.1 ms of weight streaming at 2x width).

    The recurrent state lives in static buffers owned by the graph; the state object returned by a call is a handle to
    them (valid until the next call).  Passing any other state (e.g. `policy.initial_state(B)` after an episode reset)
    copies it in.  Sampling uses torch's graph-safe Philox generator, i.e. the same `rand_like` draws as eager mode.

    memory="pytree" (default): the static state is the reference's list of (mask, (K, V)) fp32 and each step ends by copying the new
    state over it.  memory="ring": the static state is a `RingState` that the step updates in place (no copy of the memory; half its
    bytes); a pytree or another RingState passed in is copied into it, and every call returns that RingState.

    envs=E (with memory="ring"): asynchronous rollouts.  `state` is a RingState of E environments, and a call steps any k of them,
    1 <= k <= batch_size: `step(obs_k, first_k, step.state.rows(idx))` with len(idx) = k.  The call pads its static buffers to batch_size
    rows with inert rows (-1, zero frames, first False), so one graph per `stochastic` serves every subset without a host sync, and
    returns the view with the first k rows of the outputs.  It takes only views of its own `state`: install a state with
    `step.state.load_(...)` or `step.state.rows(idx).load_(...)`.

    In the batch-invariant mode (`set_batch_invariant`) a graph computes every row as the eager B = 1 step computes it, and a ring samples
    with the keys of `state.steps`, which the graph advances.  A pytree graph's stochastic call takes `noise_keys` (B, 2) as `act` does.
    Graphs are keyed on the mode and the seed: toggling either captures again."""

    def __init__(self, policy: "MinecraftAgentPolicy", batch_size: int, pdl: bool = False, memory: str = "pytree",
                 envs: Optional[int] = None):
        if memory not in ("pytree", "ring"):
            raise ValueError(f"GraphedAct: memory must be 'pytree' or 'ring' (got {memory!r})")
        if envs is not None and (memory != "ring" or envs < 1):
            raise ValueError(f"GraphedAct: envs={envs} needs memory='ring' and at least one environment")
        self.policy = policy
        self.pdl = pdl
        self.memory = memory
        self.envs = envs
        cfg = policy.net.cfg
        dev = policy.net.final_ln.weight.device
        B, self.B = batch_size, batch_size
        H, W = cfg.img_shape[0], cfg.img_shape[1]
        self.img = torch.zeros((B, H, W, 3), dtype=torch.uint8, device=dev)
        self.first = torch.zeros((B,), dtype=torch.bool, device=dev)
        self.noise_keys = torch.zeros((B, 2), dtype=torch.int64, device=dev)  # a pytree graph's keys in the batch-invariant mode
        if envs is not None:
            self.state = RingState.zeros(policy, envs)
            self.state._alloc_row_off()
            self.idx = torch.full((B,), -1, dtype=torch.int32, device=dev)
            self._view = RingRows(self.state, self.idx, [-1] * B)  # what the graph steps: the rows in self.idx
        elif memory == "ring":
            self.state = RingState.zeros(policy, B)
        else:
            self.state = [(torch.zeros((B, 1, cfg.maxlen), dtype=torch.bool, device=dev),
                           (torch.zeros((B, cfg.maxlen, cfg.hidsize), dtype=F32, device=dev),
                            torch.zeros((B, cfg.maxlen, cfg.hidsize), dtype=F32, device=dev))) for _ in range(cfg.n_layers)]
        self._held = self._layouts()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):  # warm-up outside capture (lazy function attributes, allocator pools)
            for _ in range(2):  # (a view: inert rows only)
                policy.act({"img": self.img}, self.first, self.state if envs is None else self._view, noise_keys=self._keys_arg(True))
            if memory == "ring" and envs is None:  # the warm-up stepped the ring in place: back to the empty state
                for buf in self.state.k + self.state.v + self.state.mask + [self.state.off] + [x for x in [self.state.steps] if x is not None]:
                    buf.zero_()
        torch.cuda.current_stream(dev).wait_stream(side)
        self.graphs = {}

    def _layouts(self):
        """What a captured graph reads through RAW device pointers: the kernel-layout weight copies and the de-normalisation scalars, as
        the policy holds them now (it rebuilds a stale one here, OUTSIDE any capture: they must not live in a graph's pool).  A copy
        re-laid out in place by `refresh_weights` stays the same object, and the graph reads its new values."""
        pol = self.policy
        return pol.net.prepared(), pol._heads_prepared(), pol._denorm.get()

    def _keys_arg(self, stochastic: bool):
        return self.noise_keys if self.policy.batch_invariant and self.memory == "pytree" and stochastic else None

    def _capture(self, stochastic: bool):
        if self.policy.batch_invariant and self.memory == "ring":
            self.state._alloc_steps()  # (outside the capture: the graph advances it in place)
        g = torch.cuda.CUDAGraph()
        # optional programmatic dependent launch: with the attribute the next kernel is scheduled while the previous one drains
        # (csrc/common.cuh pdl_sync).  Measured neutral for this graph (0.953 vs 0.957 ms), hence off by default.
        nat.lib().vpt_set_pdl(1 if self.pdl else 0)
        try:
            with torch.cuda.graph(g):
                state = self.state if self.envs is None else self._view
                ac, st, res = self.policy.act({"img": self.img}, self.first, state, stochastic=stochastic, return_pd=True,
                                              noise_keys=self._keys_arg(stochastic))
                if self.memory == "pytree":
                    for (m_in, (k_in, v_in)), (m_out, (k_out, v_out)) in zip(self.state, st):  # roll the state inside the graph
                        m_in.copy_(m_out)
                        if k_in.shape[1] > 0:
                            ops.copy_rows2(k_out, v_out, 0, k_in, v_in, 0, k_in.shape[1])  # K and V in one launch
        finally:
            nat.lib().vpt_set_pdl(0)
        self.graphs[self._key(stochastic)] = (g, ac, res)
        return self.graphs[self._key(stochastic)]

    def _replay(self, stochastic: bool):
        held = self._layouts()
        if any(a is not b for a, b in zip(held, self._held)):  # a copy was rebuilt since capture (a load, an optimizer step): re-capture
            self.graphs = {}
            self._held = held
        g, ac, res = self.graphs.get(self._key(stochastic)) or self._capture(stochastic)
        g.replay()
        return ac, res

    def _key(self, stochastic: bool):
        # a ring given per-row offsets (copied in from a ring that has them) runs other kernels than the graph captured without them; the
        # batch-invariant mode runs other kernels, samples under its seed, and advances the ring's `steps` through its address
        key = stochastic, self.memory == "ring" and self.state.row_off is not None
        pol = self.policy
        if not pol.batch_invariant:
            return key
        steps = self.state.steps.data_ptr() if self.memory == "ring" and self.state.steps is not None else None
        return key + (pol.noise_seed, steps)

    def _check_invariant(self, stochastic: bool, noise_keys):
        """The batch-invariant mode's refusals of `act` (its T = 1 and fp32 rules, `noise_keys`), before any copy."""
        pol = self.policy
        pol._invariant_call(1, False)
        pol._check_noise_keys(self.B, self.state if self.memory == "ring" else None, stochastic, noise_keys)

    def _call_rows(self, obs, first, view, stochastic: bool, return_pd: bool, noise_keys=None):
        """envs=E: step the k environments of `view` as rows 0..k-1 of the graph, inert rows after them."""
        if not isinstance(view, RingRows) or view.ring is not self.state:
            raise ValueError("GraphedAct(envs=E) steps views of its own ring, `step.state.rows(idx)`; install other states with "
                             "`step.state.load_` or `step.state.rows(idx).load_`")
        k, B = len(view), self.B
        if k > B:
            raise ValueError(f"GraphedAct: a view of {k} rows for a graph of batch size {B}")
        if obs["img"].shape[0] != k or first.shape[0] != k:
            raise ValueError(f"GraphedAct: {obs['img'].shape[0]} frames and {first.shape[0]} `first` flags for a view of {k} rows")
        self._check_invariant(stochastic, noise_keys)
        self.idx[:k].copy_(view.idx)
        self.img[:k].copy_(obs["img"])
        self.first[:k].copy_(first)
        if k < B:
            self.idx[k:].fill_(-1)
            self.img[k:].zero_()
            self.first[k:].zero_()
        ac, res = self._replay(stochastic)
        out = {"log_prob": res["log_prob"][:k], "vpred": res["vpred"][:k]}
        if return_pd:
            out["pd"] = {n: x[:k] for n, x in res["pd"].items()}
        return {n: x[:k] for n, x in ac.items()}, view, out

    @torch.no_grad()
    def __call__(self, obs, first, state_in, stochastic: bool = True, taken_action=None, return_pd: bool = False, noise_keys=None):
        if taken_action is not None:
            raise NotImplementedError("GraphedAct: taken_action is only supported by the eager act()")
        if self.envs is not None:
            return self._call_rows(obs, first, state_in, stochastic, return_pd, noise_keys)
        if isinstance(state_in, RingRows):
            raise ValueError("GraphedAct: a view of a ring needs GraphedAct(..., memory='ring', envs=E)")
        self._check_invariant(stochastic, noise_keys)
        if noise_keys is not None:
            self.noise_keys.copy_(noise_keys)
        self.img.copy_(obs["img"])
        self.first.copy_(first)
        if state_in is not self.state and self.memory == "ring":
            self.state.load_(state_in)
        elif state_in is not self.state:
            for (m_in, (k_in, v_in)), (m, (k, v)) in zip(self.state, state_in):
                if m is None:
                    m_in.zero_()  # lib/masked_attention.py:75-76: None == all-False
                else:
                    m_in.copy_(m)
                k_in.copy_(k)
                v_in.copy_(v)
        ac, res = self._replay(stochastic)
        out = {"log_prob": res["log_prob"], "vpred": res["vpred"]}
        if return_pd:
            out["pd"] = res["pd"]
        return ac, self.state, out
