"""Training steps of `MinecraftAgentPolicy` (behavioural cloning, RL fine-tuning) and `InverseActionPolicy`: forward with a tape, the
loss, and a hand-written backward through the same CUDA ops the forward uses -- no autograd graph.  Gradients land in `param.grad`
(fp32, reference parameter layout), so `parallel.FlatAdamDP` (one NCCL all-reduce over the flat gradient bucket + one fused Adam
launch) finishes the step.

The three trainers share one path and differ only in the loss:

    _taped_forward        the inference kernels, recording what the backward needs
    loss                  the loss and d loss / d logits, bf16 [N][ld_logits] with one column block per `_head_layers()` entry
                            BCTrainer   -mean log p(demonstrated action)                        (behavioural_cloning.py:101-123)
                            RLTrainer   clipped policy gradient + value-head MSE + KL penalty    (the value head is one more column)
                            IDMTrainer  -mean sum over sub-actions log p(action)                  (factored heads)
    _backward_from_dlog   `_heads_bwd` (the head weights, dlog -> d latent), then `_backward_from_dlat`: final_ln [-> lastlayer],
                          the transformer, img_process.linear, dense, the ImpalaCNN and, for the IDM, its conv3d pre-stage

The ImpalaCNN's activations are nearly all of a call's tape.  With `recompute_frames` (the trainers' constructors, `set_autograd`) the
forward keeps only the CNN's output and the backward re-runs the CNN chunk by chunk (`_recompute_cnn`), back-propagating through each
chunk before making the next; without it the forward's tape is the one chunk.

Only the parameters that require grad when the forward runs train (`_grad_plan`): a frozen parameter gets no gradient (its `.grad` is
left as it is), its weight-side work (`wgrad`, the norms' column sums, d b_nd, the head columns) is not done, and the backward stops at
the lowest unit of `_grad_units` that needs a gradient, without that unit's input gradient.  The forward records only what that backward
reads: with the ImpalaCNN frozen no per-stack activation at all, so the stored tape no longer bounds a call's frames.  With every
parameter trainable the same kernels run in the same order as without the rule.

The differentiable forward (`set_autograd`, `_AutogradRunner` at the end of this file) runs the same taped forward and enters the same
backward at dlog (any loss over pd / vpred, through `ops.log_softmax_bwd`) or at d latent (a bare network); its gradients go to a sink
that hands them back to autograd instead of `param.grad`.

What each layer type needs (u = gamma * n + beta is the normalised layer input, n = (x - mean) * rstd):

    NormConv / NormLinear   dz = dout * [out > 0]              ReLU (residual convs keep their branch output r for this)
                            du = dz (*) W^T                    the forward conv / GEMM kernel on flipped / transposed weights
                            dW = dz^T (*) u                    `wgrad`: wgmma GEMM over the pixel / token dimension
                            dgamma, dbeta = sum du*n, sum du   `col_sums`
                            dx = rstd * (gamma*du - mean(gamma*du) - n * mean(gamma*du*n))      `group_sums` + `norm_bwd_apply`
    max-pool, first conv, attention, softmax heads: their own backward kernels (see include/vpt_b200.h).

The KV memory carried in `state_in` is detached exactly like behavioural_cloning.py:111 (`tree_map(lambda x: x.detach())`),
and `value_head.*` receives no gradient from the BC loss (None in the reference: the BC loss never touches it).  Only the differentiable
forward with `state_grad` (`set_autograd(True, state_grad=True)`) carries gradients through it: `_backward_from_dlat` then takes the
gradient wrt each layer's state_out K / V and returns the one wrt its state_in K / V (`ops.attention_bwd_state`).
"""
import torch
import torch.distributed as dist

from . import ops
from .policy import BF16, CNN_PREFIXES, F32, FrameLatents, InverseActionPolicy, MinecraftAgentPolicy, RingRows, RingState, _dense_from_zp
from .policy import _rot  # noqa: F401  (the dgrad weight layout lived here; code that imports it from this module keeps working)


def _grad_units(net):
    """The backward's units in forward order, each a tuple of parameter-name prefixes of `net` (the heads come after the last one).  A
    unit's input gradient is computed only when a unit below it needs a gradient."""
    cfg = net.cfg
    units = [("conv3d_layer.",)] if cfg.conv3d_out is not None else []
    for i in range(len(cfg.chans)):
        s = f"img_process.cnn.stacks.{i}"
        units += [(f"{s}.firstconv.",), (f"{s}.n.",)] + [(f"{s}.blocks.{j}.conv{k}.",) for j in range(2) for k in range(2)]
    units += [("img_process.cnn.dense.",), ("img_process.linear.",)]
    for l in range(cfg.n_layers):
        b = f"recurrent_layer.blocks.{l}"
        o = f"{b}.r.orc_block"
        units += [(f"{b}.pre_r_ln.",), tuple(f"{o}.{c}_layer." for c in "qkvr"), (f"{o}.b_nd",), (f"{o}.proj_layer.",), (f"{b}.mlp0.",),
                  (f"{b}.mlp1.",)]
    if net.use_lastlayer:
        units.append(("lastlayer.",))
    units.append(("final_ln.",))
    return units


def _acc(p, g):
    """p.grad += g (allocating on first use), like autograd's accumulation."""
    g = g.reshape(p.shape)
    if p.grad is None:
        p.grad = g.to(F32).clone()
    else:
        p.grad.add_(g)


class _Trainer:
    """The machinery the trainers share: the taped forward and the backward from d logits, on the kernel-layout weights the model keeps
    (`MinecraftPolicy.prepared_backward`, `_PolicyBase._heads_prepared_backward`).  A subclass checks its policy before calling
    `_Trainer.__init__` and supplies the loss."""

    # Frames per call with `recompute_frames` (without it the stored CNN tape bounds a call first: net.cnn_chunk_frames /
    # net.idm_chunk_frames).  The CNN launches then see one chunk (at most net.cnn_chunk_frames frames, as in the inference forward);
    # every launch above the CNN takes the call's N = B*T frames as rows: the GEMMs (the dense layer over [N, (Hf+1)(Wf+1)C2], the heads
    # over [N, 8641 + ...]) as the 32-bit `vpt_gemm_args.M`, walked in 128-row tiles by a signed 32-bit TMA row coordinate; the norm,
    # elementwise, softmax and head-gradient kernels as 64-bit row / element counts; the attention and the KV-memory copies put B on a
    # grid's y axis.  So N <= 2^31 - 128 and B <= 65535; device memory (about 1 MB per frame above the CNN at 2x width) binds first.
    max_call_frames = 2 ** 31 - 128
    max_call_batch = 65535
    value_column = False  # whether the value head's output is one more column of the logits gradient (`_head_layers`)

    def __init__(self, policy, net=None, recompute_frames=None):
        """`policy` may be None with `net` given: a bare MinecraftPolicy / InverseActionNet (no heads; the differentiable forward).
        `recompute_frames`: see `BCTrainer`."""
        from .policy import check_recompute_frames

        self.policy = policy
        self.net = policy.net if net is None else net
        self.recompute_frames = check_recompute_frames(recompute_frames)
        self._sink = None  # None: gradients accumulate into `param.grad`; a dict: id(param) -> gradient (the differentiable forward)
        self.keep_tape = False   # tests: keep the last forward's tape in `self.last_tape` (tests/forced_replica.py)
        self.last_tape = None
        self.on_recompute = None  # tests: called as on_recompute(f0, f1, out, mr) with every chunk's recomputed CNN output and statistics
        self.ld_logits = (sum(lin.weight.shape[0] for lin in self._head_layers()) + 7) // 8 * 8  # columns of the logits gradient
        self._units = _grad_units(self.net)
        self._pos = {u[0]: i for i, u in enumerate(self._units)}  # a unit's first prefix -> its place in forward order
        self._train, self._lowest = frozenset(), len(self._units) + 1  # the running backward's `_grad_plan` (set from its tape)

    def _head_layers(self):
        """The linear layers whose outputs are the columns of the logits gradient `dlog` (and the rows of `heads_t`), in column order: the
        action heads, then with `value_column` the value head, so that the dgrad GEMM, `wgrad` and `col_sums` of the heads give d latent,
        dW_v and db_v as well."""
        pol = self.policy
        if pol is None:
            return []
        return [getattr(pol.pi_head, name).linear_layer for name in pol.head_specs] + ([pol.value_head.linear] if self.value_column else [])

    def _grad_plan(self, want_dmem=None, want_dimg=False):
        """What the backward of a forward starting now does, from the parameters' `requires_grad` (and, with `state_grad`, from whether
        each layer's state_in K / V gradient is wanted; `want_dimg`: the image gradient is wanted, which, like a wanted input gradient of
        unit 0, puts `lowest` below every unit) -> dict(train: ids of the parameters that train, lowest: the place in
        `_grad_units` order of the lowest unit that needs a gradient (the image: -1; the heads: len(units); nothing: len(units) + 1), stacks_from /
        blocks_from: the first CNN stack / transformer block whose activations the backward reads (their count: none), cnn: whether
        the backward enters the CNN)."""
        net, cfg, units = self.net, self.net.cfg, self._units
        train = frozenset(id(p) for p in (net if self.policy is None else self.policy).parameters() if p.requires_grad)
        names = tuple(n for n, p in net.named_parameters() if id(p) in train)
        lowest = next((i for i, u in enumerate(units) if any(n.startswith(u) for n in names)), len(units) + 1)
        if lowest > len(units) and any(id(p) in train for lin in self._head_layers() for p in (lin.weight, lin.bias)):
            lowest = len(units)
        for l, want in enumerate(want_dmem or ()):
            if want:  # the attention backward of layer l gives its state_in gradient
                lowest = min(lowest, self._pos[f"recurrent_layer.blocks.{l}.r.orc_block.b_nd"])
        if want_dimg:
            lowest = -1
        nst = len(cfg.chans)
        stacks_from = next((i for i in range(nst) if lowest <= self._pos[f"img_process.cnn.stacks.{i}.blocks.1.conv1."]), nst)
        blocks_from = next((l for l in range(cfg.n_layers) if lowest <= self._pos[f"recurrent_layer.blocks.{l}.mlp1."]), cfg.n_layers)
        if not net.use_lastlayer and lowest <= self._pos["final_ln."]:
            blocks_from = min(blocks_from, cfg.n_layers - 1)  # final_ln reads the last block's output
        return dict(train=train, lowest=lowest, stacks_from=stacks_from, blocks_from=blocks_from, cnn=stacks_from < nst, want_dimg=want_dimg)

    def _use_plan(self, tape):
        self._train, self._lowest = tape["train"], tape["lowest"]

    def _trains(self, p):
        """Whether parameter p trains in the running backward."""
        return id(p) in self._train

    def _below(self, prefix):
        """Whether a unit below the one whose first prefix is `prefix` needs a gradient, i.e. whether that unit's input gradient is needed."""
        return self._lowest < self._pos[prefix]

    def _grad(self, p, g):
        """Hands the gradient g of parameter p to the sink: `p.grad` (accumulated, `_acc`) or the dict of the differentiable forward.
        Nothing for a frozen parameter."""
        if not self._trains(p):
            return
        if self._sink is None:
            _acc(p, g)
            return
        g = g.reshape(p.shape).to(F32)
        prev = self._sink.get(id(p))
        self._sink[id(p)] = g if prev is None else prev + g

    # -- generic pieces -------------------------------------------------------------------------------------------------
    @staticmethod
    def _gemm(A, Bt, N, residual=None):
        """bf16 [M][N] = A [M][K] @ Bt[N][K]^T (+ residual)."""
        M, K = A.shape
        out = torch.empty((M, N), dtype=BF16, device=A.device)
        ops.gemm(A, Bt, out, M, N, K, residual=residual)
        return out

    def _split_grads(self, dz, u, parts):
        """The weight and bias gradients of layers whose outputs are column blocks of one GEMM: dz [rows][out] is the gradient wrt that
        output, u [rows][in] its input, and parts lists (weight, bias, r0, r1): output columns [r0, r1) are that layer's (bias None: it
        has none).  One `wgrad` (dW = dz^T u) when a weight trains and one `col_sums` when a bias does; each parameter that trains gets
        its rows."""
        dW = ops.wgrad(dz, u) if any(self._trains(w) for w, _, _, _ in parts) else None
        db = ops.col_sums(dz)[1] if any(self._trains(b) for _, b, _, _ in parts) else None
        for w, b, r0, r1 in parts:
            if self._trains(w):
                self._grad(w, dW[r0:r1])
            if self._trains(b):
                self._grad(b, db[r0:r1])

    def _norm_bwd(self, du, x, mr, gamma, rows_per_group, count, g_param, b_param, grad_map=None, zp=None, add=None, relu_x=False,
                  want_dx=True):
        """Backward of n = (x - mean) * rstd, u = gamma * n + beta given du: accumulates dgamma / dbeta into `g_param` / `b_param`
        (through `grad_map` when the kernel-side gamma has another layout), returns dx (+ add), or None without `want_dx`.
        relu_x: x is the output of a ReLU whose backward is applied to the result in the same pass."""
        if rows_per_group > 1:  # GroupNorm frames: column sums and group sums share one pass over (du, x)
            cs, ms = ops.norm_sums(du, x, mr, gamma, rows_per_group, count)
        else:
            cs = ops.col_sums(du, x, mr, rows_per_group) if self._trains(g_param) or self._trains(b_param) else None
            ms = ops.group_sums(du, x, mr, gamma, rows_per_group, count) if want_dx else None
        for p, c in ((g_param, 0), (b_param, 1)):
            if self._trains(p):
                self._grad(p, cs[c] if grad_map is None else grad_map(cs[c]))
        if not want_dx:
            return None
        return ops.norm_bwd_apply(du, x, mr, gamma, ms, rows_per_group, zp=zp, add=add, relu_x=relu_x)

    def _normed_bwd(self, pfx, P, dz, x, mr, dgrad, renorm, geom, dW_map=None, shifts=(0,), gb=None, add=None, relu_x=False):
        """Backward of the normalised layer `pfx` (z = layer(u), u = gamma * n + beta) given dz [rows][out], the gradient wrt z (ReLU
        already applied); x [rows][in] is the layer input and mr its statistics.  The layer kind supplies what differs: dgrad() -> du
        [rows][in], the forward kernel on the dgrad weight; renorm(gamma, beta) -> u; geom: the norm geometry (`_norm_bwd`'s
        rows_per_group, count, zp, grad_map); dW_map: `wgrad(dz, u, shifts)` -> the weight's shape (None: it has that shape); gb: the
        kernel-side fp32 (gamma, beta) when they are not the parameters'.  Accumulates the gradients of the parameters that train and
        returns the gradient wrt x (+ add), [rows][in], or None when no unit below needs it."""
        gam, bet, wt = P[pfx + ".norm.weight"], P[pfx + ".norm.bias"], P[pfx + ".layer.weight"]
        g32, b32 = gb or (gam.detach().float().contiguous(), bet.detach().float().contiguous())
        want_dx = self._below(pfx + ".")
        norm = want_dx or self._trains(gam) or self._trains(bet)
        du = dgrad() if norm else None
        if self._trains(wt):
            dW = ops.wgrad(dz, renorm(g32, b32).view(x.shape), shifts)
            self._grad(wt, dW if dW_map is None else dW_map(dW))
            del dW
        if not norm:
            return None
        return self._norm_bwd(du, x, mr, g32, g_param=gam, b_param=bet, add=add, relu_x=relu_x, want_dx=want_dx, **geom)

    def _normconv_bwd(self, dz, x, mr, H, W, W_rot, pfx, P, add=None, relu_x=False):
        """GroupNorm over each frame -> 3x3 conv (`_normed_bwd`): dz ZP [F, H+1, W+1, Cout], x ZP [F, H+1, W+1, Cin]; W_rot the
        rotated weight (`policy._rot`).  Returns the gradient wrt x (+ add) or None."""
        Cin, Cout = x.shape[3], dz.shape[3]
        R = x.shape[0] * (H + 1) * (W + 1)
        dx = self._normed_bwd(pfx, P, dz.view(R, Cout), x.view(R, Cin), mr,
                              dgrad=lambda: ops.conv3x3_zp(dz, W_rot, H, W, relu=0, want_stats=False)[0].view(R, Cin),
                              renorm=lambda g, b: ops.affine_norm_zp(x, mr, g, b)[0],
                              shifts=[(ky - 1) * (W + 1) + (kx - 1) for ky in range(3) for kx in range(3)],
                              dW_map=lambda dW: dW.view(Cout, 3, 3, Cin).permute(0, 3, 1, 2),  # [Cout][tap][Cin]
                              geom=dict(rows_per_group=(H + 1) * (W + 1), count=H * W * Cin, zp=(H, W, Cin)),
                              add=None if add is None else add.view(R, Cin), relu_x=relu_x)
        return None if dx is None else dx.view(x.shape)

    def _normlinear_bwd(self, dz, x, mr, Wt, pfx, P, add=None, relu_x=False):
        """LayerNorm over each row -> Linear (`_normed_bwd`): dz [rows][out], x [rows][in]; Wt the transposed weight (`policy._tr`).
        Returns the gradient wrt x (+ add) or None."""
        return self._normed_bwd(pfx, P, dz, x, mr, dgrad=lambda: self._gemm(dz, Wt, Wt.shape[0]),
                                renorm=lambda g, b: ops.affine_norm(x, mr, g, b, rows_per_group=1)[0],
                                geom=dict(rows_per_group=1, count=x.shape[1]), add=add, relu_x=relu_x)

    # -- the step ---------------------------------------------------------------------------------------------------------
    def check_call(self, img, want_dimg=False):
        """The limits of one call, checked by every entry point before any launch so that a call that cannot finish accumulates nothing:
        the bf16 mode; for the IDM at most `IDMTrainer.max_t` frames per sequence; with the stored tape (recompute_frames None) and a
        backward that enters the CNN (`_grad_plan`, want_dimg: see there) at most `net.cnn_chunk_frames` (the IDM: `net.idm_chunk_frames`)
        frames, the one CNN chunk the tape holds; otherwise `max_call_frames` frames and B <= `max_call_batch`.
        From cached latents (`FrameLatents`, no CNN tape) `max_call_frames` and `max_call_batch` hold, and ValueError is raised for latents
        the network cannot take (`MinecraftPolicy.check_latents`: shape, stale), latents that require grad, and a parameter of the CNN part
        (`img_process.cnn.*`, `conv3d_layer.*`) that requires grad: it would get no gradient."""
        net = self.net
        B, t = img.shape[:2]
        if net.precision != "bf16":
            raise NotImplementedError("training and the differentiable forward run in the bf16 mode only (set_precision('bf16'))")
        if net.cfg.conv3d_out is not None and t > IDMTrainer.max_t:
            raise NotImplementedError(f"the IDM's backward takes at most {IDMTrainer.max_t} frames per sequence (got T = {t})")
        if isinstance(img, FrameLatents):
            if img.requires_grad:
                raise ValueError("latents carry no autograd graph: there is no gradient wrt them (pass the frames for an image gradient)")
            trainable = next((n for n, p in net.named_parameters() if p.requires_grad and n.startswith(CNN_PREFIXES)), None)
            if trainable is not None:
                raise ValueError(f"a call from latents trains nothing at or below img_process.cnn.dense, but {trainable} requires grad: "
                                 "freeze the CNN part (requires_grad_(False)) or pass the frames")
            net.check_latents(img)
            if B * t > self.max_call_frames or B > self.max_call_batch:
                raise NotImplementedError(f"at most {self.max_call_frames} frames and B <= {self.max_call_batch} per call (got B = {B}, T = {t})")
            return
        if self.recompute_frames is None and self._grad_plan(want_dimg=want_dimg)["cnn"]:
            limit = net.cnn_chunk_frames if net.cfg.conv3d_out is None else net.idm_chunk_frames
            if B * t > limit:
                raise NotImplementedError(f"at most {limit} frames per call with the stored CNN tape (got B*T = {B * t}); accumulate over "
                                          "calls, pass recompute_frames (set_autograd(True, recompute_frames=...)) or freeze the CNN")
        elif B * t > self.max_call_frames or B > self.max_call_batch:
            raise NotImplementedError(f"at most {self.max_call_frames} frames and B <= {self.max_call_batch} per call (got B = {B}, T = {t})")

    def _taped_latent(self, img, first, state_in, want_dmem=None, want_dimg=False):
        """The network's inference kernels, recording what the backward needs -> (latent bf16 [N][h], latent fp32 (B,t,h), tape, state_out).
        The tape also holds the kernel-layout weights the forward used (`prep`) and those the backward will use (`wts`, `heads_t`), and
        the backward's `_grad_plan` (want_dmem, want_dimg: see there).  The caller has checked the call's limits (`check_call`)."""
        net, pol = self.net, self.policy
        if isinstance(state_in, (RingState, RingRows)):
            raise ValueError("RingState is for inference: the trainers and the differentiable forward take the pytree state")
        tape = self._grad_plan(want_dmem, want_dimg)
        if pol is not None:
            pol.refresh_weights()  # (a bare network: the getters rebuild eagerly on use)
        layers = self._head_layers()
        state_in = [(m, (k.detach(), v.detach())) for (m, (k, v)) in state_in]  # behavioural_cloning.py:111
        tape.update(stacks=[], blocks=[], wts=net.prepared_backward(), heads_t=pol._heads_prepared_backward(layers) if layers else None,
                    recompute=self.recompute_frames)
        net._tape = tape
        try:
            lat_bf16, lat_f32, state_out = net._forward_impl(img, first, state_in)
        finally:
            net._tape = None
        if tape["lowest"] > self._pos["img_process.cnn.dense."]:  # the backward stops above the dense layer, which alone reads cnn_out
            tape.update(cnn_out=None, mr_c=None)
        if self.keep_tape:
            self.last_tape = tape
        return lat_bf16, lat_f32, tape, state_out

    def _taped_forward(self, img, first, state_in, mask=None, want_dmem=None, want_dimg=False):
        """The inference kernels, recording what the backward needs -> (latent bf16, pd, vpred, tape, state_out)."""
        B, t = img.shape[:2]
        lat_bf16, _, tape, state_out = self._taped_latent(img, first, state_in, want_dmem, want_dimg)
        pd, vpred = self.policy._heads(lat_bf16, B, t, mask)
        return lat_bf16, pd, vpred, tape, state_out

    def _backward_from_dlog(self, dlog, lat_bf16, tape, B, t, upper_grads_ready):
        """Everything below the logits: the head weights (`_heads_bwd`), then `_backward_from_dlat` when a unit below the heads trains.
        dlog may be None when nothing trains."""
        dlat = None if dlog is None else self._heads_bwd(dlog, lat_bf16, tape)
        del dlog
        if dlat is not None:
            self._backward_from_dlat(dlat, tape, B, t, upper_grads_ready)
        elif upper_grads_ready is not None:
            upper_grads_ready()

    def _heads_bwd(self, dlog, lat_bf16, tape):
        """The head weights' gradients from dlog bf16 [N][ld_logits] (one column block per `_head_layers()` entry) -> d latent bf16 [N][h],
        or None when nothing below the heads trains."""
        self._use_plan(tape)
        parts, c0 = [], 0
        for lin in self._head_layers():
            parts.append((lin.weight, lin.bias, c0, c0 + lin.weight.shape[0]))
            c0 += lin.weight.shape[0]
        self._split_grads(dlog, lat_bf16, parts)
        return self._gemm(dlog, tape["heads_t"], self.net.cfg.hidsize) if self._lowest < len(self._units) else None

    def _backward_from_dlat(self, dlat, tape, B, t, upper_grads_ready, dstate=None, want_dmem=None):
        """Everything below the latent (the output of final_ln): final_ln [, lastlayer], the transformer, img_process.linear, dense, the
        ImpalaCNN and, for the IDM, the conv3d pre-stage.  dstate: None or per layer None / (dk, dv), the gradient wrt that layer's
        state_out K / V; want_dmem: None or per layer whether its state_in gradient is wanted.  Returns per layer (dmem_k, dmem_v) or None.
        Each stage runs only while a unit at or below it needs a gradient (`_grad_plan`); `upper_grads_ready` is called once, before the
        CNN or, when the backward does not enter it, at its end.  With the image gradient wanted (`_grad_plan`'s want_dimg) it is left in
        tape["dimg"], fp32 [N, H, W, 3] on the uint8 scale."""
        self._use_plan(tape)
        net = self.net
        cfg = net.cfg
        wts = tape["wts"]
        P = dict(net.named_parameters())
        h = cfg.hidsize
        # ---------------- final_ln (plain norm) on lastlayer's output, or on relu(recurrent output) without lastlayer ----------------
        # (xl, z_last, x0, xd and the convs' h are ReLU outputs that feed a norm: their ReLU backward rides on that norm's apply pass)
        dx = None
        if self._lowest <= self._pos["final_ln."]:
            if net.use_lastlayer:
                x, mr = tape["xl"], tape["mr_xl"]
            else:  # lib/policy.py:389-392: the last block's z, relu fused into its epilogue
                x, mr = tape["blocks"][-1]["z"], tape["blocks"][-1]["mr_z"]
            fg = P["final_ln.weight"]
            dx = self._norm_bwd(dlat, x, mr, fg.detach().float().contiguous(), 1, h, fg, P["final_ln.bias"], relu_x=True,
                                want_dx=self._below("final_ln."))
        if dx is not None and net.use_lastlayer:
            dx = self._normlinear_bwd(dx, tape["z_last"], tape["mr_zl"], wts["last_t"], "lastlayer", P, relu_x=True)
        # ---------------- transformer blocks, last to first ----------------
        dmem = [None] * cfg.n_layers
        for l in reversed(range(cfg.n_layers)):
            if dx is None:
                break
            dx, dmem[l] = self._block_bwd(l, dx, tape["blocks"][l], tape["first_u8"], wts["layers"][l], P, B, t,
                                          dstate=None if dstate is None else dstate[l], want_dmem=bool(want_dmem and want_dmem[l]))
        # ---------------- img_process.linear, dense ----------------
        dz = None if dx is None else self._normlinear_bwd(dx, tape["xd"], tape["mr_d"], wts["linear_t"], "img_process.linear", P, relu_x=True)
        dcnn = None if dz is None else self._dense_bwd(dz, tape, wts, P)
        if upper_grads_ready is not None:
            upper_grads_ready()
        # ---------------- ImpalaCNN, last stack to first, chunk by chunk (last chunk first) ----------------
        # The stored tape is the one-chunk case: its per-stack activations come from the forward.  With `recompute` every chunk's are made
        # again from the frames and the forward's weights, used, and dropped before the next chunk.  (No chunk when the CNN is frozen.)
        # The gradient wrt the CNN input (`_cnn_bwd`) is the image gradient for the agent's fused first conv, and for the IDM the gradient
        # wrt the conv3d output, which its own backward takes to the weights and, when wanted, to the image; each chunk writes its frames'.
        chunks = tape["cnn_chunks"]
        if not chunks:  # the CNN is frozen, or the call came from cached latents (no frames): the backward ends above the dense layer
            return dmem
        frames = tape["frames"]
        dimg = None
        if tape["want_dimg"] and len(chunks) > 1:
            dimg = torch.empty((frames.shape[0], *frames.shape[1:3], 3), dtype=F32, device=frames.device)
        for f0, f1 in reversed(chunks):
            ct = tape if tape["recompute"] is None else self._recompute_cnn(tape, f0, f1, t)
            dx3 = self._cnn_bwd(dcnn[f0:f1], ct, wts, P)
            del ct
            di = None
            if cfg.conv3d_out is None:
                di = dx3
            elif dx3 is not None:
                # the IDM's conv3d pre-stage: kernel weights are W_ref[C][c][dt] / 255 laid out [C][dt][c] (policy._Prepared)
                C3 = cfg.conv3d_out
                w3, b3 = net.conv3d_layer.layer.weight, net.conv3d_layer.layer.bias
                if self._trains(w3) or self._trains(b3):
                    dW3, db3 = ops.conv3d_t5_bwd(frames[f0:f1].view((f1 - f0) // t, t, *frames.shape[1:]), dx3, C3)
                    self._grad(w3, (dW3 / 255.0).view(C3, 5, 3).permute(0, 2, 1))
                    self._grad(b3, db3)
                if tape["want_dimg"]:
                    di = ops.conv3d_t5_dimg(dx3, tape["prep"].conv3d[0], (f1 - f0) // t, t, *frames.shape[1:3])
            del dx3
            if di is not None:
                if dimg is None:
                    dimg = di
                else:
                    dimg[f0:f1] = di
            del di
        del dcnn
        if tape["want_dimg"]:
            tape["dimg"] = dimg
        return dmem

    def _recompute_cnn(self, tape, f0, f1, t):
        """The forward of CNN chunk [f0, f1) again, in the training layout with the kernel-layout weights the forward used (tape["prep"]),
        recording what `_cnn_bwd` needs (the stacks from tape["stacks_from"] on) -> that chunk's tape.  The kernels are deterministic, so this is the forward's chunk bit for bit."""
        net = self.net
        cfg = net.cfg
        frames = tape["frames"][f0:f1]
        img = frames if cfg.conv3d_out is None else frames.view((f1 - f0) // t, t, *frames.shape[1:])
        Hf, Wf = cfg.final_hw
        out = torch.empty((f1 - f0, Hf + 1, Wf + 1, cfg.chans[-1]), dtype=BF16, device=frames.device)
        stacks = []
        with torch.no_grad():
            _, mr = net._cnn_chunk(img, tape["prep"], out, train=True, stacks=stacks, record_from=tape["stacks_from"])
        if self.on_recompute is not None:
            self.on_recompute(f0, f1, out, mr)
        return dict(stacks=stacks, prep=tape["prep"], frames=frames)

    def _dense_bwd(self, dz, tape, wts, P):
        """The dense layer: LayerNorm -> Linear over the CNN output's ZP rows (`_normed_bwd`), with its kernel-side gamma / beta and weight
        columns in ZP order (`policy._dense_to_zp`); its gradients go back to the reference's order.  Returns the gradient wrt the CNN
        output, ZP [N, Hf+1, Wf+1, C2], or None."""
        cfg = self.net.cfg
        Hf, Wf = cfg.final_hw
        C2 = cfg.chans[-1]
        N = dz.shape[0]
        Kd = (Hf + 1) * (Wf + 1) * C2
        x, mr = tape["cnn_out"].view(N, Kd), tape["mr_c"]
        unperm = lambda v: _dense_from_zp(v, cfg)
        dx = self._normed_bwd("img_process.cnn.dense", P, dz, x, mr, dgrad=lambda: self._gemm(dz, wts["dense_t"], Kd),
                              renorm=lambda g, b: ops.affine_norm(x, mr, g, b, rows_per_group=1)[0],
                              geom=dict(rows_per_group=1, count=Hf * Wf * C2, zp=(Hf, Wf, C2), grad_map=unperm), dW_map=unperm,
                              gb=(wts["dense_g"], wts["dense_b"]))
        return None if dx is None else dx.view(N, Hf + 1, Wf + 1, C2)

    def _block_bwd(self, l, dzo, S, first_u8, W, P, B, t, dstate=None, want_dmem=False):
        """Backward of lib/util.py:193-211 (see policy.MinecraftPolicy._block for the forward in the same notation) -> (d block input,
        (dmem_k, dmem_v) or None).  dstate: None or (dk, dv), the gradient wrt the layer's state_out K / V (either None); want_dmem: return
        the gradient wrt its state_in K / V (lib/xf.py:366-391 builds the memory with cat and slicing, so autograd reaches it).  The d block
        input is None when no unit below the block needs it; the backward then stops at the lowest unit of the block that needs a gradient."""
        cfg = self.net.cfg
        h, heads, maxlen = cfg.hidsize, cfg.heads, cfg.maxlen
        b = f"recurrent_layer.blocks.{l}"
        o = f"{b}.r.orc_block"
        N = B * t
        nr = 10 * heads
        trains = self._trains
        dz = dzo  # (last block: z is relu(..) (lib/policy.py:211 fused into its epilogue); the norm backward above already masked dzo)
        # mlp1: z = y + hmid W1^T + b1
        dh = self._gemm(dz, W["mlp1_t"], h * cfg.pointwise_ratio) if self._below(f"{b}.mlp1.") else None
        self._split_grads(dz, S["hmid"], [(P[f"{b}.mlp1.layer.weight"], P[f"{b}.mlp1.layer.bias"], 0, h)])
        if dh is None:
            return None, None
        # mlp0: hmid = relu(LN(y) W0^T)
        dzh = ops.relu_mask(dh, S["hmid"])
        del dh
        dy = self._normlinear_bwd(dzh, S["y"], S["mr_y"], W["mlp0_t"], f"{b}.mlp0", P, add=dz)
        del dzh
        if dy is None:
            return None, None
        # proj: y = xhat + a Wp^T + bp
        da = self._gemm(dy, W["proj_t"], h) if self._below(f"{o}.proj_layer.") else None
        self._split_grads(dy, S["a"], [(P[f"{o}.proj_layer.weight"], P[f"{o}.proj_layer.bias"], 0, h)])
        if da is None:
            return None, None
        # attention: gradients wrt q | k | v | R side by side (one buffer = one dgrad GEMM + one wgrad GEMM for all four)
        causal = cfg.mask_style == "clipped_causal"
        dqkvr = torch.zeros((N, cfg.kcat), dtype=BF16, device=dy.device)
        dmem = None
        if causal and (dstate is not None or want_dmem):  # the KV memory is in the graph (the differentiable forward's state_grad)
            db_nd, dmem = ops.attention_bwd_state(S["q"], S["full_k"], S["full_v"], S["R"], P[f"{o}.b_nd"].detach().float().contiguous(), first_u8,
                                                  S["smask"], da, dqkvr, B, t, maxlen, heads, dstate=dstate, want_dmem=want_dmem)
        elif causal:
            db_nd = ops.attention_bwd(S["q"], S["full_k"], S["full_v"], S["R"], P[f"{o}.b_nd"].detach().float().contiguous(), first_u8, S["smask"],
                                      da, dqkvr, B, t, maxlen, heads)
        else:  # mask "none" (IDM): q | k | v only; R meets an empty band (b_nd is (10, 0)), so its parameters get exact zeros
            ops.attention_bwd(S["q"], S["full_k"], S["full_v"], None, None, None, None, da, dqkvr, B, t, 0, heads, causal=False)
            db_nd = torch.zeros_like(P[f"{o}.b_nd"], dtype=F32) if trains(P[f"{o}.b_nd"]) else None
        self._grad(P[f"{o}.b_nd"], db_nd)
        if not self._below(f"{o}.b_nd"):
            return None, dmem
        # q | k | v | r: one dgrad GEMM and one wgrad GEMM for the four (r only where the mask has a band)
        dxhat = self._gemm(dqkvr, W["qkvr_t"], h, residual=dy) if self._below(f"{o}.q_layer.") else None
        parts = [(P[f"{o}.q_layer.weight"], P[f"{o}.q_layer.bias"], 0, h), (P[f"{o}.k_layer.weight"], None, h, 2 * h),
                 (P[f"{o}.v_layer.weight"], None, 2 * h, 3 * h)]
        if causal:
            parts.append((P[f"{o}.r_layer.weight"], P[f"{o}.r_layer.bias"], 3 * h, 3 * h + nr))
        self._split_grads(dqkvr, S["xhat"], parts)
        if not causal:
            for p in (P[f"{o}.r_layer.weight"], P[f"{o}.r_layer.bias"]):
                if trains(p):
                    self._grad(p, torch.zeros_like(p, dtype=F32))
        if dxhat is None:
            return None, dmem
        # pre_r_ln (plain norm of the block input)
        g = P[f"{b}.pre_r_ln.weight"]
        dx = self._norm_bwd(dxhat, S["x"], S["mr_x"], g.detach().float().contiguous(), 1, h, g, P[f"{b}.pre_r_ln.bias"],
                            relu_x=(l == 0), want_dx=self._below(f"{b}.pre_r_ln."))  # block 0's input is relu(img_process.linear)
        return dx, dmem

    def _cnn_bwd(self, dout, tape, wts, P):
        """Backward of lib/impala_cnn.py:187-195; `dout` is the gradient wrt the last stack's output (ZP).  Returns the gradient wrt the
        CNN input when a unit below needs it: when stack 0's first conv is a normalised one (the IDM) the gradient wrt the conv3d output,
        ReLU backward applied; for the fused first conv the image gradient (fp32 [F, H, W, 3]), when it is wanted; else None.  Stops at the
        lowest unit that needs a gradient."""
        cfg = self.net.cfg
        pfx = "img_process.cnn"
        dx = dout
        for i in reversed(range(len(cfg.chans))):
            rec = tape["stacks"][i]
            s = f"{pfx}.stacks.{i}"
            H, W = rec["H_in"] // 2, rec["W_in"] // 2
            C = cfg.chans[i]
            R = dx.shape[0] * (H + 1) * (W + 1)
            for j in (1, 0):
                blk = rec["blocks"][j]
                x_in = rec["blocks"][j - 1]["x"] if j == 1 else rec["x0"]
                mr_in = rec["blocks"][j - 1]["mr"] if j == 1 else rec["mr0"]
                # x_out = x_in + relu(conv1(GN(h)));  h = relu(conv0(GN(x_in)))
                dz1 = ops.relu_mask(dx, blk["r"])
                dz0 = self._normconv_bwd(dz1, blk["h"], blk["mrh"], H, W, wts["stacks"][i]["convs"][2 * j + 1], f"{s}.blocks.{j}.conv1", P,
                                         relu_x=True)
                del dz1
                if dz0 is None:
                    return None
                dx = self._normconv_bwd(dz0, x_in, mr_in, H, W, wts["stacks"][i]["convs"][2 * j], f"{s}.blocks.{j}.conv0", P, add=dx)
                del dz0
                if dx is None:
                    return None
            # x0 = GN_n(y1) (plain norm)
            g = P[f"{s}.n.weight"]
            dy1 = self._norm_bwd(dx.view(R, C), rec["y1"].view(R, C), rec["mr1"], g.detach().float().contiguous(), (H + 1) * (W + 1), H * W * C,
                                 g, P[f"{s}.n.bias"], zp=(H, W, C), want_dx=self._below(f"{s}.n."))
            if dy1 is None:
                return None
            dy1 = dy1.view(rec["y1"].shape)
            if i == 0 and not cfg.first_conv_norm:
                st = tape["prep"].stacks[0]  # (the weights the forward used)
                wp, bp = P[f"{s}.firstconv.layer.weight"], P[f"{s}.firstconv.layer.bias"]
                if self._trains(wp) or self._trains(bp):
                    dWk, db = ops.firstconv_bwd(tape["frames"], st["fc_w"], st["fc_b"], dy1, C)
                    # kernel weights are W[c0][ky][kx][c] / 255 (lib/policy.py:44 folded in)
                    self._grad(wp, (dWk / 255.0).view(C, 3, 3, 3).permute(0, 3, 1, 2))
                    self._grad(bp, db)
                return ops.firstconv_dimg(tape["frames"], st["fc_w"], st["fc_b"], dy1, C) if self._lowest < 0 else None
            dfull = ops.maxpool3s2_bwd(dy1, rec["full"])  # includes the ReLU in front of the pool
            del dy1
            # (IDM stack 0: the input is the ReLU output of the conv3d pre-stage; its ReLU backward rides on this norm's apply pass)
            dx = self._normconv_bwd(dfull, rec["x_in"], rec["mr_in"], rec["H_in"], rec["W_in"], wts["stacks"][i]["first"],
                                    f"{s}.firstconv", P, relu_x=(i == 0))
            del dfull
            if dx is None:
                return None
        return dx


class BCTrainer(_Trainer):
    """Behavioural-cloning step of `MinecraftAgentPolicy` (behavioural_cloning.py:101-123):
    `loss, state_out = trainer.loss_and_grad(img, first, state_in, actions)` accumulates d loss / d param into `.grad`.

        loss = -(1 / (B*T)) * sum_{b,t} sum_heads log_softmax(logits_head / temperature)[action]      (lib/action_head.py:176-184)

    recompute_frames=None keeps the ImpalaCNN's activations from the forward for the backward: at most `net.cnn_chunk_frames` (2048)
    frames per call, and at 2x width 20.7 MiB per frame with its backward workspace (H100, README).  recompute_frames=F (a positive int) keeps only the CNN's output: the forward
    runs the CNN in chunks of F frames (at most `net.cnn_chunk_frames`) and the backward re-runs each chunk's forward before
    back-propagating through it.  That costs one more CNN forward per call and allows `max_call_frames` frames per call (e.g. B = 128,
    T = 128 in one call at 2x width); the gradients are those of the stored tape.

    Parameters with requires_grad=False when the call starts are frozen: their `.grad` is left as it is, their weight-side work is skipped
    and the backward stops at the lowest unit that trains.  With the whole ImpalaCNN (`img_process.cnn.*`) frozen the forward keeps no
    CNN activation, so a call is bounded by `max_call_frames` instead of the stored tape, and `upper_grads_ready` fires at the end of the
    backward.  With nothing trainable the call returns the loss and state_out and runs no backward.

    `img` may instead be cached latents (`FrameLatents`, `policy.encode(img)`, with the CNN part frozen): the call then runs no CNN, forward
    or backward, and gives the loss, state_out and gradients of the same call from `img` with the CNN frozen, bit for bit.  Its limits are
    `max_call_frames` and `max_call_batch`; `recompute_frames` has nothing to recompute and is ignored for such a call.  The same holds for
    `RLTrainer` and `IDMTrainer` (see INTEGRATION.md, "cached latents").
    """

    def __init__(self, policy: MinecraftAgentPolicy, recompute_frames=None):
        if not isinstance(policy, MinecraftAgentPolicy):
            raise TypeError(f"{type(self).__name__} trains a MinecraftAgentPolicy (behavioural_cloning.py:54-62)")
        cfg = policy.net.cfg
        if cfg.conv3d_out is not None or cfg.first_conv_norm or cfg.mask_style != "clipped_causal":
            raise NotImplementedError(f"{type(self).__name__}: only the causal policy models are trained by the reference")
        super().__init__(policy, recompute_frames=recompute_frames)

    def _check_heads(self):
        """Every head must have a single sub-action.  Checked before the forward: nothing is accumulated into .grad by a call that
        cannot finish."""
        pol = self.policy
        if any(getattr(pol.pi_head, name).linear_layer.weight.shape[0] != n for name, (shape, n) in pol.head_specs.items()):
            raise NotImplementedError(f"{type(self).__name__}: heads with several sub-actions are not trained by the reference")

    def loss_and_grad(self, img, first, state_in, actions, upper_grads_ready=None):
        """`upper_grads_ready()` is called once every gradient except those of `img_process.cnn.stacks.*` is final (the ImpalaCNN
        backward, most of the step's time, is still to come): the hook for `FlatAdamDP.reduce_async`."""
        self._check_heads()
        self.check_call(img)
        lat_bf16, pd, _, tape, state_out = self._taped_forward(img, first, state_in)
        loss, dlog = self._bc_dlog(pd, actions, img.shape[0] * img.shape[1], want_dlog=tape["lowest"] <= len(self._units))
        self._backward_from_dlog(dlog, lat_bf16, tape, img.shape[0], img.shape[1], upper_grads_ready)
        return loss, state_out

    def _bc_dlog(self, pd, actions, N, want_dlog=True):
        """The BC loss -mean log p(action) over the N frames and its gradient wrt the logits, bf16 [N][ld_logits] (None without
        `want_dlog`: nothing trains)."""
        pol = self.policy
        hp = pol._heads_prepared()
        dlog = torch.zeros((N, self.ld_logits), dtype=BF16, device=pol.net.final_ln.weight.device) if want_dlog else None
        scale = 1.0 / (pol.temperature * N)
        logp = None
        for name, (shape, n) in pol.head_specs.items():
            idx = actions[name].reshape(N).to(torch.int64)
            lp = ops.gather_logprob(pd[name].reshape(N, n), idx)
            logp = lp if logp is None else logp + lp
            if want_dlog:
                ops.softmax_bwd(pd[name].reshape(N, n), idx, scale, dlog, hp["cols"][name][0])
        return -logp.sum() / N, dlog


class RLTrainer(BCTrainer):
    """RL fine-tuning step of `MinecraftAgentPolicy`: a clipped policy-gradient (PPO) loss, the value head's loss and a KL penalty to the
    frozen pretrained policy, with the shared hand-written backward.  Over the N = B*T frames of one call:

        lp      = sum over heads of log pi(a)                     (get_logprob_of_action, lib/policy.py:271-279)
        ratio   = exp(lp - old_logprob)
        L_pi    = -mean min(ratio * A, clamp(ratio, 1 - clip, 1 + clip) * A)
        L_v     = mean (vpred - normalizer(returns))^2            (ScaledMSEHead.loss in training mode, lib/scaled_mse_head.py:37-43:
                                                                   the EWMA normaliser is updated with this batch first)
        L_kl    = mean KL(pi_ref || pi)                           (get_kl_of_action_dists(pd_ref, pd), lib/policy.py:281-285)
        H       = mean H(pi)                                      (pi_head.entropy(pd), lib/action_head.py:186-194)
        loss    = L_pi + vf_coef * L_v + kl_coef * L_kl - ent_coef * H

    `loss, state_out = trainer.loss_and_grad(img, first, state_in, actions, old_logprob, advantages, returns, pd_ref, vf_coef=..,
    kl_coef=.., ent_coef=..)` accumulates d loss / d param into `.grad` (the value head included) and updates the normaliser once in place;
    under `torch.distributed` its batch statistics are all-reduced first, so every rank holds the normaliser of the global batch.
    `old_logprob`, `advantages` and `returns` are fp32 (B, T), `returns` in the denormalised space; `pd_ref` is what the frozen
    reference policy's forward returns for the same frames (None only with kl_coef == 0).  `ent_coef` (default 0) is the entropy bonus;
    with 0 the step runs exactly as without the term.  `trainer.stats` holds 0-d device tensors pi_loss, vf_loss, kl_ref, clipfrac and
    entropy (H) of the last call.  With ent_coef == 0 the step runs the kernels of the step without the term and does not compute the
    entropy: `stats["entropy"]` (or `.get("entropy")`) computes it, one read of the call's log-probs, when first read; the next call frees
    those log-probs, so read it before then (`_RLStats`).  Hand every parameter with `requires_grad` to the optimizer (the three
    normaliser tensors have none).  `recompute_frames` as in `BCTrainer`."""

    ewma_beta = 0.99999  # NormalizeEwma's default (lib/normalize_ewma.py:9; per_element_update=False, norm over (B, T))
    value_column = True   # the value head trains with the action heads

    def __init__(self, policy: MinecraftAgentPolicy, recompute_frames=None):
        super().__init__(policy, recompute_frames=recompute_frames)
        self.stats = None

    def loss_and_grad(self, img, first, state_in, actions, old_logprob, advantages, returns, pd_ref=None, *, vf_coef, kl_coef, clip=0.2,
                      ent_coef=0.0, upper_grads_ready=None):
        """`upper_grads_ready` as in `BCTrainer.loss_and_grad`."""
        pol = self.policy
        B, t = img.shape[:2]
        N = B * t
        for name, x in (("old_logprob", old_logprob), ("advantages", advantages), ("returns", returns)):
            if x.dtype != F32 or tuple(x.shape) != (B, t) or x.device != img.device:
                raise ValueError(f"RLTrainer: {name} must be fp32 {(B, t)} on {img.device} (got {x.dtype} {tuple(x.shape)} on {x.device})")
        if pd_ref is None and kl_coef != 0:
            raise ValueError("RLTrainer: kl_coef != 0 needs pd_ref, the frozen reference policy's action distributions")
        if pd_ref is not None:
            for name, (shape, n) in pol.head_specs.items():
                if pd_ref[name].dtype != F32 or pd_ref[name].numel() != N * n:
                    raise ValueError(f"RLTrainer: pd_ref[{name!r}] must be fp32 with {N} x {n} log-probs (got {tuple(pd_ref[name].shape)})")
        self._check_heads()
        self.check_call(img)
        if isinstance(self.stats, _RLStats):  # the last call's unread statistics: free their log-probs before this call's forward
            self.stats.release()
        lat_bf16, pd, vpred, tape, state_out = self._taped_forward(img, first, state_in)
        loss, dlog = self._rl_dlog(pd, vpred, actions, old_logprob, advantages, returns, pd_ref, vf_coef, kl_coef, clip, N, ent_coef)
        self._backward_from_dlog(dlog, lat_bf16, tape, B, t, upper_grads_ready)
        return loss, state_out

    def _rl_dlog(self, pd, vpred, actions, old_logprob, advantages, returns, pd_ref, vf_coef, kl_coef, clip, N, ent_coef=0.0):
        pol = self.policy
        hp = pol._heads_prepared()
        dlog = torch.zeros((N, self.ld_logits), dtype=BF16, device=vpred.device)
        idx, logp = {}, None
        for name, (shape, n) in pol.head_specs.items():
            idx[name] = actions[name].reshape(N).to(torch.int64).contiguous()
            lp = ops.gather_logprob(pd[name].reshape(N, n), idx[name])
            logp = lp if logp is None else logp + lp
        c, pi_loss, clipped = ops.ppo_coef(logp, old_logprob.reshape(N).contiguous(), advantages.reshape(N).contiguous(), clip)
        kl = ent = None
        for name, (shape, n) in pol.head_specs.items():
            q = None if pd_ref is None else pd_ref[name].reshape(N, n)
            if ent_coef:  # the fused entropy bonus; it also gives the entropy per row
                kl, ent = ops.rl_head_bwd_ent(pd[name].reshape(N, n), idx[name], c, q, kl_coef / N, ent_coef / N, 1.0 / pol.temperature, dlog,
                                              hp["cols"][name][0], kl, ent)
            else:
                kl = ops.rl_head_bwd(pd[name].reshape(N, n), idx[name], c, q, kl_coef / N, 1.0 / pol.temperature, dlog, hp["cols"][name][0], kl)
        # value head: the normaliser sees the global batch (one 2-element all-reduce under data parallelism), then the scaled MSE
        ret = returns.reshape(N).contiguous()
        sums = ops.ewma_sums(ret)
        count = N
        if dist.is_available() and dist.is_initialized():
            dist.all_reduce(sums)
            count = N * dist.get_world_size()
        nz = pol.value_head.normalizer
        sq = ops.value_bwd(vpred.reshape(N), ret, sums, count, nz.running_mean, nz.running_mean_sq, nz.debiasing_term, self.ewma_beta,
                           2.0 * vf_coef / N, dlog, hp["ntot"])
        stats = dict(pi_loss=pi_loss.mean(), vf_loss=sq.mean(), kl_ref=kl.mean(), clipfrac=clipped.mean())
        loss = stats["pi_loss"] + vf_coef * stats["vf_loss"] + kl_coef * stats["kl_ref"]
        if ent_coef:
            stats["entropy"] = ent.mean()
            loss = loss - ent_coef * stats["entropy"]
            self.stats = stats
        else:
            self.stats = _RLStats(stats, entropy=lambda: pol.pi_head.entropy(pd).mean())
        return loss, dlog


class _RLStats(dict):
    """`RLTrainer.stats`: a dict of 0-d device tensors, with the statistics the step did not compute (the entropy when ent_coef == 0) made
    on first read by their function, which holds the call's log-probs until then.  `stats[key]`, `stats.get(key)` and `key in stats` see
    such a statistic; iteration, `len` and `items()` show it once it has been read.  The trainer's next call drops what is still unread
    (`release`), so the held log-probs never overlap that call's own."""

    def __init__(self, stats, **lazy):
        super().__init__(stats)
        self._lazy = lazy

    def __missing__(self, key):
        if key not in self._lazy:
            raise KeyError(key)
        self[key] = v = self._lazy.pop(key)()
        return v

    def __contains__(self, key):
        return super().__contains__(key) or key in self._lazy

    def get(self, key, default=None):
        return self[key] if key in self else default

    def release(self):
        self._lazy.clear()


class IDMTrainer(_Trainer):
    """Training step of the inverse dynamics model (`InverseActionPolicy`, lib/policy.py:342-467) with the shared hand-written backward:
    `loss, state_out = trainer.loss_and_grad(img, first, state_in, actions)` accumulates d loss / d param into `.grad`.

        loss = -(1 / (B*T)) * sum_{b,t} sum_heads sum_sub-actions log_softmax(logits / temperature)[action]

    `actions` = {"buttons": int (B,T,20), "camera": int (B,T,2)}, the layout `InverseActionPolicy.predict` returns.  The backward runs
    heads -> final_ln on relu(recurrent output) -> the unmasked transformer blocks -> img_process.linear -> dense -> ImpalaCNN ->
    the conv3d pre-stage.  Which parameters get which gradient follows the reference's autograd: `lastlayer.*` gets None (its
    output is discarded, lib/policy.py:390-391); `r_layer.*` gets zeros and `b_nd` an empty (10, 0) gradient (R meets an empty band).

    One call holds whole sequences (the temporal conv needs the neighbouring frames).  With recompute_frames=None it holds at most
    `net.idm_chunk_frames` (512) frames, i.e. B = 4 at T = 128: the training forward keeps the whole CNN tape of one call.  With
    recompute_frames=F the CNN runs, and is re-run in the backward, in chunks of F frames rounded down to whole sequences (at least one,
    at most `net.idm_chunk_frames`), and a call may hold `max_call_frames` frames (as in `BCTrainer`).  Batches also accumulate over calls
    (`.grad` accumulates, as with BCTrainer).  T <= 128, bf16 only.  `first` and the state do nothing with mask "none": the state stays
    (None, (B,0,h), (B,0,h))."""

    max_t = 128  # frames per sequence the unmasked attention backward supports

    def __init__(self, policy: InverseActionPolicy, recompute_frames=None):
        if not isinstance(policy, InverseActionPolicy):
            raise TypeError("IDMTrainer trains an InverseActionPolicy (lib/policy.py:406-467)")
        cfg = policy.net.cfg
        if cfg.conv3d_out is None or cfg.mask_style != "none" or cfg.maxlen != 0:
            raise NotImplementedError("IDMTrainer: needs the IDM configuration (conv3d pre-stage, attention mask 'none', no KV memory)")
        if cfg.timesteps is not None and cfg.timesteps > self.max_t:
            raise NotImplementedError(f"IDMTrainer: the unmasked attention backward supports chunks of at most {self.max_t} frames")
        super().__init__(policy, recompute_frames=recompute_frames)

    @staticmethod
    def optimizer_params(policy):
        """The parameters to hand to `FlatAdamDP`, in the order that makes its bucket split like BC's: `conv3d_layer.*` first, then the
        policy's parameters in registration order without `lastlayer.*` (no gradient, lib/policy.py:390-391).  The gradients that are
        final when `upper_grads_ready` fires then form the bucket slice [opt.offset_of(net.img_process.cnn.dense.norm.weight), opt.n):
        the conv3d pre-stage, whose gradient comes last, is registered after the transformer and would otherwise sit inside it."""
        named = [(n, p) for n, p in policy.named_parameters() if not n.startswith("net.lastlayer.")]
        return [p for n, p in named if n.startswith("net.conv3d_layer.")] + [p for n, p in named if not n.startswith("net.conv3d_layer.")]

    def loss_and_grad(self, img, first, state_in, actions, upper_grads_ready=None):
        """`upper_grads_ready()` is called once every gradient except those of `img_process.cnn.stacks.*` and `conv3d_layer.*` is final
        (the CNN backward, most of the step's time, is still to come): the hook for `FlatAdamDP.reduce_async`.  Build the optimizer from
        `optimizer_params(policy)` so that those final gradients are one contiguous bucket slice."""
        B, t = img.shape[:2]
        self.check_call(img)
        lat_bf16, pd, _, tape, state_out = self._taped_forward(img, first, state_in)
        loss, dlog = self._idm_dlog(pd, actions, B * t)
        self._backward_from_dlog(dlog, lat_bf16, tape, B, t, upper_grads_ready)
        return loss, state_out

    def _idm_dlog(self, pd, actions, N):
        """The loss -mean sum log p(action) over the N frames and every sub-action, and its gradient wrt the logits, bf16 [N][ld_logits]
        (one launch per factored head)."""
        pol = self.policy
        hp = pol._heads_prepared()
        dlog = torch.zeros((N, self.ld_logits), dtype=BF16, device=pol.net.final_ln.weight.device)
        scale = 1.0 / (pol.temperature * N)
        logp = None
        for name, (shape, n) in pol.head_specs.items():
            c0, width = hp["cols"][name]
            groups = width // n
            idx = actions[name].reshape(N, groups).to(torch.int64)
            logp = ops.softmax_nll_bwd_grouped(pd[name].reshape(N, groups, n), idx, scale, dlog, c0, lp=logp)
        return -logp.sum() / N, dlog


# -- the differentiable forward (`set_autograd`) ------------------------------------------------------------------------------
class _AutogradRunner(_Trainer):
    """The shared taped forward and backward behind `loss.backward()`: `_PolicyBase.set_autograd(True)` (or `MinecraftPolicy.set_autograd`)
    makes the forward an autograd `Function` whose backward turns the upstream gradients of its outputs into one gradient per parameter.

        agent policy   outputs pd (one fp32 tensor per head) and vpred;  d pd -> `ops.log_softmax_bwd` -> dlog columns, d vpred -> the
                       value head's column; then `_heads_bwd` and `_backward_from_dlat`
        IDM policy     outputs pd
        bare network   outputs the latent;  d latent -> `_backward_from_dlat`

    Gradients go to a dict (`_Trainer._grad` with a sink) and are returned to autograd, which accumulates them into `.grad`.  A parameter
    that only feeds outputs the loss does not touch gets None, as in the reference's autograd.

    With `state_grad` (`set_autograd(True, state_grad=True)`, models with a KV memory) the state_in K / V of every layer are inputs of the
    `Function` too and the state_out K / V extra outputs, so a loss on a later call reaches this one through the memory (truncated BPTT:
    the caller detaches the state every k calls).  The backward then also takes d state_out and returns d state_in
    (`ops.attention_bwd_state`); a call whose own outputs get no gradient but whose state_out does runs the same backward from a zero d
    latent."""

    def __init__(self, module):
        from .policy import _PolicyBase

        pol = module if isinstance(module, _PolicyBase) else None
        self.value_column = pol is not None and pol.has_value_head  # vpred is an output
        super().__init__(pol, None if pol is not None else module)
        self.module = module

    def state_grad(self):
        """Whether this module's differentiable forward carries gradients through the KV memory (`set_autograd(.., state_grad=True)`;
        nothing changes for a model without memory, maxlen = 0: the IDM)."""
        return bool(getattr(self.module, "_state_grad", False)) and self.net.cfg.maxlen > 0

    def check_state_in(self, state_in):
        """Without `state_grad`, a state_in that requires grad is refused: no gradient flows through the KV memory across calls."""
        if self.state_grad():
            return
        for _, (k, v) in state_in:
            if k.requires_grad or v.requires_grad:
                raise ValueError("differentiable forward: state_in must not require grad -- gradients do not flow through the KV memory "
                                 "across calls; detach the state (behavioural_cloning.py:109-111) or opt in with "
                                 "set_autograd(True, state_grad=True)")

    def run(self, img, first, state_in, mask=None):
        """-> (outputs, state_out): outputs attached to the graph (pd per head [+ vpred], or the latent); state_out detached, or with
        `state_grad` its K / V attached (state_mask is a plain bool tensor either way).  An `img` that requires grad is one more input (its
        fp32 copy, `policy.frames_f32`, so that autograd casts the gradient back to the leaf's dtype) whose gradient the backward returns."""
        from .policy import frames_f32

        self.recompute_frames = self.module._recompute_frames  # set_autograd(.., recompute_frames=..)
        self.check_call(img, want_dimg=img.requires_grad)
        self.check_state_in(state_in)
        params = [p for p in self.module.parameters()]
        sg = self.state_grad()
        kv = [x for _, (k, v) in state_in for x in (k, v)] if sg else []
        ig = img.requires_grad
        if ig:
            img = frames_f32(img)
        box = dict(img=img, first=first, state_in=state_in, mask=mask, state_grad=sg, img_grad=ig)
        outs = _TapedForward.apply(self, box, *params, *kv, *((img,) if ig else ()))
        outs = (outs,) if isinstance(outs, torch.Tensor) else outs
        if not sg:
            return outs, box["state_out"]
        n = len(outs) - len(kv)
        kvo = outs[n:]
        return outs[:n], [(m, (kvo[2 * l], kvo[2 * l + 1])) for l, (m, _) in enumerate(box["state_out"])]

    def forward_outputs(self, box):
        """Runs the taped forward -> (output tensors, tape)."""
        img = box["img"]
        B, t = img.shape[:2]
        # with state_grad, a state_in K / V that requires grad is an input whose gradient the backward returns
        want = [k.requires_grad or v.requires_grad for _, (k, v) in box["state_in"]] if box["state_grad"] else None
        ig = box["img_grad"]
        if self.policy is None:
            lat_bf16, lat_f32, tape, state_out = self._taped_latent(img, box["first"], box["state_in"], want, ig)
            outs = (lat_f32,)
        else:
            mask = box["mask"]
            lat_bf16, pd, vpred, tape, state_out = self._taped_forward(img, box["first"], box["state_in"], mask, want, ig)
            outs = tuple(pd.values()) + ((vpred,) if vpred is not None else ())
            masks = {}
            for name, (shape, n) in self.policy.head_specs.items():
                if mask is not None and mask.get(name) is not None:
                    m = mask[name].to(device=img.device, dtype=torch.bool).expand(pd[name].shape)
                    masks[name] = m.reshape(B * t, -1).contiguous()
            tape["head_masks"] = masks
        tape.update(lat=lat_bf16, B=B, t=t)
        box["state_out"] = state_out
        return outs, tape

    def backward_grads(self, tape, outs, grads, dstate=None, want_dmem=None):
        """The upstream gradients of the outputs -> ({id(param): gradient} (parameters absent from it get None), per layer d state_in
        (dmem_k, dmem_v) or None).  dstate / want_dmem as in `_backward_from_dlat` (the `state_grad` case)."""
        B, t = tape["B"], tape["t"]
        N = B * t
        sink = {}
        self._sink = sink
        h = self.net.cfg.hidsize
        try:
            if all(g is None for g in grads):  # only the state_out feeds the loss: no head gradient, a zero d latent
                return sink, self._backward_from_dlat(torch.zeros((N, h), dtype=BF16, device=tape["lat"].device), tape, B, t, None, dstate,
                                                      want_dmem)
            if self.policy is None:
                return sink, self._backward_from_dlat(grads[0].reshape(N, -1).to(BF16).contiguous(), tape, B, t, None, dstate, want_dmem)
            pol = self.policy
            hp = pol._heads_prepared()
            dlog = torch.zeros((N, self.ld_logits), dtype=BF16, device=tape["lat"].device)
            unused = []
            for i, (name, (shape, n)) in enumerate(pol.head_specs.items()):
                lin = getattr(pol.pi_head, name).linear_layer
                if grads[i] is None:
                    unused.append(lin)
                    continue
                c0, width = hp["cols"][name]
                g = grads[i].reshape(N, width).to(F32).contiguous()
                ops.log_softmax_bwd(outs[i].reshape(N, width), g, 1.0 / pol.temperature, dlog, c0, width // n, tape["head_masks"].get(name))
            if pol.has_value_head:
                gv = grads[len(pol.head_specs)]
                if gv is None:
                    unused.append(pol.value_head.linear)
                else:
                    dlog[:, hp["ntot"]] = gv.reshape(N).to(BF16)  # d vpred: the value head's column (a strided copy of N values)
            dlat = self._heads_bwd(dlog, tape["lat"], tape)
            del dlog
            dmem = [None] * self.net.cfg.n_layers if dlat is None else self._backward_from_dlat(dlat, tape, B, t, None, dstate, want_dmem)
            for lin in unused:
                sink.pop(id(lin.weight), None)
                sink.pop(id(lin.bias), None)
            return sink, dmem
        finally:
            self._sink = None


def _aligned_f32(x):
    """x as a contiguous, 16-byte aligned fp32 tensor (the layout the state-gradient kernel reads)."""
    x = x.to(F32).contiguous()
    return x if x.data_ptr() % 16 == 0 else x.clone()


class _TapedForward(torch.autograd.Function):
    """forward(runner, box, *params[, *state K / V][, img]): the taped forward; the tape lives in ctx until the backward frees it.  The
    parameters are inputs (saved, so that an in-place change before the backward raises torch's version-check error); the kernel-layout
    weights the forward used are in the tape, so the backward never re-lays out newer parameters.  With `box["state_grad"]` the state_in
    K / V of every layer follow the parameters as inputs, and the state_out K / V follow the outputs.  With `box["img_grad"]` the fp32
    frames are the last input and the backward returns the image gradient for them."""

    @staticmethod
    def forward(ctx, runner, box, *inputs):
        ctx.set_materialize_grads(False)
        outs, tape = runner.forward_outputs(box)
        n_params = len(inputs) - (2 * len(box["state_in"]) if box["state_grad"] else 0) - (1 if box["img_grad"] else 0)
        ctx.runner, ctx.tape, ctx.n_params, ctx.n_outs = runner, tape, n_params, len(outs)
        ctx.img_shape = tuple(box["img"].shape) if box["img_grad"] else None
        ctx.save_for_backward(*inputs[:n_params], *outs)
        if box["state_grad"]:
            outs = outs + tuple(x for _, (k, v) in box["state_out"] for x in (k, v))
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *grads):
        if torch.is_grad_enabled():
            raise NotImplementedError("the differentiable forward has no double backward (create_graph=True)")
        if ctx.tape is None:  # (checked first: torch has freed the saved tensors too)
            raise RuntimeError("the differentiable forward's tape was freed by an earlier backward: a graph can be back-propagated once "
                               "(with state_grad, detach the state or call backward once per window)")
        saved = ctx.saved_tensors  # (raises if a parameter or an output was modified in place since the forward)
        tape, ctx.tape = ctx.tape, None
        params, outs = saved[:ctx.n_params], saved[ctx.n_params:]
        dstate = want_dmem = None
        if len(grads) > ctx.n_outs:  # state_grad: per layer d state_out K / V, and whether d state_in K / V is wanted
            gs, need = grads[ctx.n_outs:], ctx.needs_input_grad[2 + ctx.n_params:]
            L = len(gs) // 2
            dstate = [None if gs[2 * l] is None and gs[2 * l + 1] is None else (gs[2 * l], gs[2 * l + 1]) for l in range(L)]
            dstate = [None if d is None else tuple(None if x is None else _aligned_f32(x) for x in d) for d in dstate]
            want_dmem = [need[2 * l] or need[2 * l + 1] for l in range(L)]
        sink, dmem = ctx.runner.backward_grads(tape, outs, grads[:ctx.n_outs], dstate, want_dmem)
        dimg = tape.get("dimg")
        del tape
        mods = list(ctx.runner.module.parameters())
        res = [sink.get(id(p)) if ctx.needs_input_grad[2 + i] else None for i, p in enumerate(mods)]
        if want_dmem is not None:
            need = ctx.needs_input_grad[2 + ctx.n_params:]
            for l, d in enumerate(dmem):
                res += [d[0] if d is not None and need[2 * l] else None, d[1] if d is not None and need[2 * l + 1] else None]
        if ctx.img_shape is not None:
            res.append(dimg.view(ctx.img_shape) if ctx.needs_input_grad[-1] else None)
        return (None, None) + tuple(res)
