"""TEST-ONLY float64 references of the forward kernels, and the forward call shapes of the released models.

The references are the oracle's own layer functions (oracle/vpt_oracle.py: `fanin_conv`, `cnn_basic_block`, `fanin_linear`,
`conv3d_stage`, ...) run in float64 on whatever device the inputs are on, with the weights of a reference-schema state dict.  They
restate the unfused layers -- GroupNorm / LayerNorm materialised, then the convolution or linear -- so a kernel fed the product's
fold tables (`policy._Prepared`: `_fold_conv`, `_fold_conv2`, `_fold_linear`, `_class_taps`, `_dense_to_zp`) is held to the
layer it replaces, not to an emulation of the same fold (tests/emu_ops.py).  `forward_shapes` derives every shape from the model
config, so the tests follow the model when it changes."""
import torch
import torch.nn.functional as F

import vpt_b200
import vpt_oracle as O
from common import make_policy, perturb
from video_pre_training_b200.policy import NBASIS, MinecraftPolicy, NetConfig

F64 = torch.float64
BF16 = torch.bfloat16
MODELS = ["1x", "2x", "3x", "idm"]


# ---------------------------------------------------------------------------------------------------------------------
# shapes
# ---------------------------------------------------------------------------------------------------------------------
def model_kwargs(width):
    return vpt_b200.idm_net_kwargs() if width == "idm" else vpt_b200.policy_kwargs(width)


def forward_shapes(width):
    """The call shapes the inference forward (policy.py, `_forward_impl`) reaches for the released model `width` (1x / 2x / 3x / idm)."""
    cfg = NetConfig(**model_kwargs(width))
    H, W, cin = cfg.img_shape
    stacks = []
    for i, c in enumerate(cfg.chans):  # the first conv runs at the stack's input size; the pool halves it for the blocks
        stacks.append(dict(H=H, W=W, Cin=cin, C=c, fused_first=i == 0 and not cfg.first_conv_norm))
        H, W, cin = H // 2, W // 2, c
    Hf, Wf = cfg.final_hw
    assert (H, W) == (Hf, Wf)
    kd = (Hf + 1) * (Wf + 1) * cfg.chans[-1]
    h, heads = cfg.hidsize, cfg.heads
    causal = cfg.mask_style == "clipped_causal"
    space = vpt_b200.idm_action_space() if width == "idm" else vpt_b200.minecraft_action_space()
    cols, c0 = [], 0
    for name, sp in space.items():
        n = sp.eltype.n
        cnt = 1
        for s in sp.shape:
            cnt *= s
        cols.append((name, c0, n, cnt))  # cnt sub-actions of n classes side by side
        c0 += n * cnt
    linears = dict(dense=(cfg.cnn_outsize, kd), linear=(h, cfg.cnn_outsize), mlp0=(h * cfg.pointwise_ratio, h), mlp1=(h, h * cfg.pointwise_ratio),
                   proj=(h, h))
    if width != "idm":
        linears["lastlayer"] = (h, h)
    return dict(
        cfg=cfg, stacks=stacks, firstconv=cfg.chans[0] if stacks[0]["fused_first"] else None, conv3d=cfg.conv3d_out,
        dense=(Hf, Wf, cfg.chans[-1], kd), h=h, heads=heads, maxlen=cfg.maxlen, t=cfg.timesteps, causal=causal,
        qkvr=3 * h + (NBASIS * heads if causal else 0), head_cols=cols, ntot=c0, ld_logits=(c0 + 7) // 8 * 8, linears=linears,
        chunk=MinecraftPolicy.idm_chunk_frames if width == "idm" else MinecraftPolicy.cnn_chunk_frames,
    )


# ---------------------------------------------------------------------------------------------------------------------
# weights: a perturbed policy of the model's config (the net's state-dict keys, no "net." prefix)
# ---------------------------------------------------------------------------------------------------------------------
def make_model(width, seed=0):
    """The perturbed agent policy (MinecraftAgentPolicy, or InverseActionPolicy for the IDM) of `width` on the CPU, and the state dict of
    its net (fp32, keys without the "net." prefix)."""
    if width == "idm":
        torch.manual_seed(seed)
        pol = vpt_b200.InverseActionPolicy(vpt_b200.idm_action_space(), dict(temperature=2.0), model_kwargs(width))
        perturb(pol)
    else:
        pol, _, _ = make_policy(model_kwargs(width), seed=seed)
    return pol, {k: v.detach() for k, v in pol.net.state_dict().items()}


class SD64(dict):
    """A state dict whose entries are converted to float64 on `device` when first read (the refs touch a few layers only)."""

    def __init__(self, sd, device):
        super().__init__()
        self.src, self.device = sd, device

    def __contains__(self, k):
        return k in self.src

    def __getitem__(self, k):
        if not dict.__contains__(self, k):
            dict.__setitem__(self, k, self.src[k].to(self.device, F64))
        return dict.__getitem__(self, k)

    def get(self, k, default=None):
        return self[k] if k in self.src else default


# ---------------------------------------------------------------------------------------------------------------------
# ZP helpers (ZP = [F, H+1, W+1, C] with a zero last row / column)
# ---------------------------------------------------------------------------------------------------------------------
def nchw(zp):
    return zp[:, :-1, :-1, :].to(F64).permute(0, 3, 1, 2)


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1)


def stats(v, zp=False):
    """float64 (mean, rstd) per frame (zp: of the interior of a ZP tensor) or per row of what a kernel stored: [G][2]."""
    if zp:
        v = v[:, :-1, :-1, :]
    x = v.to(F64).reshape(v.shape[0], -1)
    return torch.stack([x.mean(1), 1 / torch.sqrt(x.var(1, unbiased=False) + 1e-5)], 1)


def chan_sums(y_zp, parts):
    """Per-channel (sum, sumsq) partials of the interior of ZP y as the pool kernels hand them to vpt_norm2_fold: fp32 [F][parts][C][2],
    one partial per band of rows (the float64 sums rounded once)."""
    yi = y_zp[:, :-1, :-1, :].to(F64)
    Fn, H, W, C = yi.shape
    b = yi.reshape(Fn, parts, H // parts * W, C)
    return torch.stack([b.sum(2), (b * b).sum(2)], -1).float()


# ---------------------------------------------------------------------------------------------------------------------
# references (float64, the oracle's layers)
# ---------------------------------------------------------------------------------------------------------------------
def firstconv_pool(img_u8, sd, p):
    """stack 0: u8 / 255 -> fanin_conv (bias, no norm) -> max_pool2d(3, 2, 1), NHWC float64 (and the pre-pool map)."""
    x = img_u8.to(F64).permute(0, 3, 1, 2) / 255.0
    full = O.fanin_conv(x, sd, p + ".firstconv")
    return nhwc(F.max_pool2d(full, 3, 2, 1))


def conv(x_zp, sd, p):
    """fanin_conv: GroupNorm(1) on the input -> conv3x3 -> ReLU, NHWC float64."""
    return nhwc(O.fanin_conv(nchw(x_zp), sd, p))


def maxpool(full_zp):
    return nhwc(F.max_pool2d(nchw(full_zp), 3, 2, 1))


def block(x_zp, sd, p, n=None):
    """cnn_basic_block on x (n: the stack's post-pool GroupNorm prefix, applied first, as the folded block 0 of inference does).
    Returns (conv0 output, block output), NHWC float64."""
    x = nchw(x_zp)
    if n is not None:
        x = F.group_norm(x, 1, sd[n + ".weight"], sd[n + ".bias"], eps=1e-5)
    taps = {}
    y = O.cnn_basic_block(x, sd, p, taps)
    return nhwc(taps[p + ".conv0"]), nhwc(y)


def conv3d(img_u8, sd, p):
    """IDM pre-stage: u8 / 255 -> conv3d (5, 1, 1) per sequence -> ReLU; [B*T, H, W, C] float64."""
    y = O.conv3d_stage(img_u8.to(F64) / 255.0, sd, p)
    return y.reshape(-1, *y.shape[2:])


def linear(x, sd, p, relu=True):
    return O.fanin_linear(x.to(F64), sd, p, relu=relu)


def plain_linear(x, sd, p, bias=True):
    """F.linear with the weight / bias `p`.weight / `p`.bias (the attention's projections and the heads: no norm, no ReLU)."""
    return F.linear(x.to(F64), sd[p + ".weight"], sd[p + ".bias"] if bias else None)


# ---------------------------------------------------------------------------------------------------------------------
# plain-NHWC forms (the fp32-parity mode, video-pre-training_b200/precise.py: fp32 [F, H, W, C] activations, no ZP pads)
# ---------------------------------------------------------------------------------------------------------------------
def conv_nhwc(x, sd, p):
    """fanin_conv on plain NHWC x: [GroupNorm(1)] -> conv3x3 -> ReLU, NHWC float64."""
    return nhwc(O.fanin_conv(x.to(F64).permute(0, 3, 1, 2), sd, p))


def maxpool_nhwc(x):
    return nhwc(F.max_pool2d(x.to(F64).permute(0, 3, 1, 2), 3, 2, 1))


def group_norm_nhwc(x, sd, p):
    """the stack's post-pool GroupNorm(1) `p` (.weight / .bias) on plain NHWC x, float64."""
    return nhwc(F.group_norm(x.to(F64).permute(0, 3, 1, 2), 1, sd[p + ".weight"], sd[p + ".bias"], eps=1e-5))


def layer_norm(x, sd, p):
    return F.layer_norm(x.to(F64), (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps=1e-5)


def dense_from_nhwc(x, Hf, Wf, C):
    """rows of the final activation flattened H, W, C (as the fp32 mode feeds the dense layer) -> flattened C, H, W (the reference's order)."""
    return x.reshape(x.shape[0], Hf, Wf, C).permute(0, 3, 1, 2).reshape(x.shape[0], -1)
