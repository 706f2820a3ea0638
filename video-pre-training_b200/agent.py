"""Caller-side mirror of the reference's `agent.py` (the boundary's caller, SURVEY rows f-2 / f-3 / f-4):

    MineRLAgent(env=None, device="cuda", policy_kwargs=None, pi_head_kwargs=None)
        .load_weights(path) / .reset() / .get_action(minerl_obs)            agent.py:106-206

plus the two pieces of arithmetic that sit right before and after the policy in a rollout:

* frame ingest  -- `resize_frames`: bilinear uint8 resize on the GPU, bit-exact with `cv2.resize(..., INTER_LINEAR)`
  (agent.py:100-103, inverse_dynamics_model.py:54-59) via `vpt_resize_bilinear_u8`;
* action codec  -- `ActionCodec`: joint (buttons 8641 x camera 121) indices <-> factored MineRL actions and the mu-law camera
  (de)quantiser, as closed-form / table lookups (lib/action_mapping.py:120-234, lib/actions.py:48-178), vectorised
  (the reference's `from_factored` is a per-row Python loop).

Everything here is re-stated from the reference's behaviour (tests compare against the live reference where it is
available); nothing needs gym, gym3 or MineRL to be installed.
"""
import itertools
from collections import OrderedDict

import numpy as np
import torch

from . import _native as nat
from . import policy as _policy
from .types import minecraft_action_space

# lib/actions.py:21-33
BUTTONS = ["attack", "back", "forward", "jump", "left", "right", "sneak", "sprint", "use", "drop", "inventory"] + \
          [f"hotbar.{i}" for i in range(1, 10)]
# lib/action_mapping.py:19-28 (+ the camera meta action, :126-127); itertools.product order: the LAST group varies fastest
BUTTON_GROUPS = OrderedDict(
    hotbar=["none"] + [f"hotbar.{i}" for i in range(1, 10)], fore_back=["none", "forward", "back"],
    left_right=["none", "left", "right"], sprint_sneak=["none", "sprint", "sneak"], use=["none", "use"],
    drop=["none", "drop"], attack=["none", "attack"], jump=["none", "jump"], camera=["none", "camera"])

AGENT_RESOLUTION = (128, 128)                       # agent.py:14
ACTION_TRANSFORMER_KWARGS = dict(camera_binsize=2, camera_maxval=10, camera_mu=10, camera_quantization_scheme="mu_law")  # agent.py:40-45


class ActionCodec:
    """CameraHierarchicalMapping(n_camera_bins=11) + ActionTransformer(**ACTION_TRANSFORMER_KWARGS) as lookup tables."""

    def __init__(self, n_camera_bins=11, camera_binsize=2, camera_maxval=10, camera_mu=10, camera_quantization_scheme="mu_law"):
        self.n_bins, self.null_bin = n_camera_bins, n_camera_bins // 2
        self.binsize, self.maxval, self.mu, self.scheme = camera_binsize, camera_maxval, camera_mu, camera_quantization_scheme
        sizes = [len(v) for v in BUTTON_GROUPS.values()]
        self.n_buttons_joint = int(np.prod(sizes)) + 1      # + "inventory" (lib/action_mapping.py:128)
        self.inventory_idx = self.n_buttons_joint - 1
        # joint index -> 20 factored buttons, camera-meta-off flag (lib/action_mapping.py:151-177)
        self.idx_to_factored = np.zeros((self.n_buttons_joint, len(BUTTONS)), dtype=np.int64)
        self.idx_camera_off = np.zeros(self.n_buttons_joint, dtype=bool)
        for i, comb in enumerate(itertools.product(*BUTTON_GROUPS.values())):
            for choice in comb[:-1]:
                if choice != "none":
                    self.idx_to_factored[i, BUTTONS.index(choice)] = 1
            self.idx_camera_off[i] = comb[-1] != "camera"
        self.idx_to_factored[self.inventory_idx, BUTTONS.index("inventory")] = 1
        self.strides = np.array([int(np.prod(sizes[k + 1:])) for k in range(len(sizes))], dtype=np.int64)
        self.camera_null_idx = self.null_bin * n_camera_bins + self.null_bin
        self.null_buttons_idx = 0                            # every group "none" (lib/action_mapping.py:146-148)

    # ---- joint -> factored (lib/action_mapping.py:215-225) ------------------------------------------------------------
    def to_factored(self, ac):
        b = np.asarray(ac["buttons"]).squeeze(-1)
        c = np.asarray(ac["camera"]).squeeze(-1)
        cam = np.stack([c // self.n_bins, c % self.n_bins], axis=-1).astype(np.int64)
        cam[self.idx_camera_off[b]] = self.null_bin
        return dict(buttons=self.idx_to_factored[b], camera=cam)

    # ---- factored -> joint (lib/action_mapping.py:193-213, :65-99), vectorised ---------------------------------------------
    def from_factored(self, ac):
        btn = np.asarray(ac["buttons"]).astype(np.int64)
        cam = np.asarray(ac["camera"]).astype(np.int64)
        assert btn.ndim == 2 and cam.ndim == 2
        B = lambda name: btn[:, BUTTONS.index(name)]

        def group(names, mutual_cancel=False):
            """index of the chosen option of a mutually exclusive group; the LATER button wins when several are pressed,
            and forward+back / left+right pressed together mean neither (lib/action_mapping.py:85-99)."""
            pressed = np.stack([B(n) for n in names], axis=-1) != 0
            if mutual_cancel:
                pressed = pressed & ~pressed.all(axis=-1, keepdims=True)
            choice = np.zeros(btn.shape[0], dtype=np.int64)
            for k in range(len(names)):
                choice = np.where(pressed[:, k], k + 1, choice)
            return choice

        choices = [group([f"hotbar.{i}" for i in range(1, 10)]), group(["forward", "back"], True), group(["left", "right"], True),
                   group(["sprint", "sneak"]), group(["use"]), group(["drop"]), group(["attack"]), group(["jump"])]
        cam_null = (cam == self.null_bin).all(axis=1)
        choices.append(np.where(cam_null, 0, 1))
        joint = sum(c * s for c, s in zip(choices, self.strides))
        inv = B("inventory") == 1
        joint = np.where(inv, self.inventory_idx, joint)
        cam_idx = np.where(inv, self.camera_null_idx, cam[:, 0] * self.n_bins + cam[:, 1])
        return dict(buttons=joint[:, None], camera=cam_idx[:, None])

    # ---- camera quantiser (lib/actions.py:82-102) -----------------------------------------------------------------------
    def discretize_camera(self, xy):
        xy = np.clip(xy, -self.maxval, self.maxval)
        if self.scheme == "mu_law":
            xy = xy / self.maxval
            xy = np.sign(xy) * (np.log(1.0 + self.mu * np.abs(xy)) / np.log(1.0 + self.mu)) * self.maxval
        return np.round((xy + self.maxval) / self.binsize).astype(np.int64)

    def undiscretize_camera(self, pq):
        xy = pq * self.binsize - self.maxval
        if self.scheme == "mu_law":
            xy = xy / self.maxval
            xy = np.sign(xy) * (1.0 / self.mu) * ((1.0 + self.mu) ** np.abs(xy) - 1.0) * self.maxval
        return xy

    # ---- on-device versions (csrc/codec.cuh): tables built here with the formulas above, look-ups on the GPU -------------------
    def _device_tables(self, device):
        device = torch.device(device)
        t = getattr(self, "_dev_tables", None)
        if t is None or t["device"] != device:
            bins = np.arange(self.n_bins)
            cam_lut = self.undiscretize_camera(bins).astype(np.float64)            # lib/actions.py:96-102, one entry per bin
            # bin thresholds of discretize_camera: thr[k] = the smallest float64 x with discretize(x) >= k + 1, found by bisection on the
            # host formula itself (monotone), so the device binning `#{k: x >= thr[k]}` reproduces numpy's log / round bit for bit
            thr = np.empty(self.n_bins - 1, dtype=np.float64)
            for k in range(self.n_bins - 1):
                lo, hi = -float(self.maxval), float(self.maxval)
                assert self.discretize_camera(np.array(lo)) <= k < self.discretize_camera(np.array(hi))
                while True:
                    mid = lo + (hi - lo) / 2
                    if mid == lo or mid == hi:
                        break
                    if self.discretize_camera(np.array(mid)) >= k + 1:
                        hi = mid
                    else:
                        lo = mid
                thr[k] = hi
            t = dict(device=device, lut_btn=torch.from_numpy(self.idx_to_factored.astype(np.uint8)).contiguous().to(device),
                     lut_cam_off=torch.from_numpy(self.idx_camera_off.astype(np.uint8)).to(device), cam_lut=torch.from_numpy(cam_lut).to(device),
                     thr=torch.from_numpy(thr).to(device), strides=torch.from_numpy(self.strides.astype(np.int64)).to(device))
            self._dev_tables = t
        return t

    def to_env_device(self, ac):
        """{"buttons": int64 (..., 1), "camera": int64 (..., 1)} device tensors (what `act` returns) -> MineRL env action dict of numpy
        arrays, == policy2env(to_factored(ac)): the look-ups run on the GPU (`vpt_codec_to_env`) and ONE (n, 22)-word tensor crosses
        to the host instead of two index tensors followed by numpy table gathers."""
        from . import ops
        b, c = ac["buttons"], ac["camera"]
        t = self._device_tables(b.device)
        lead = tuple(b.shape[:-1])
        words, bad = ops.codec_to_env(b.reshape(-1).contiguous(), c.reshape(-1).contiguous(), t["lut_btn"], t["lut_cam_off"], t["cam_lut"], self.n_bins)
        host = words.cpu().numpy()
        out = {name: host[:, i].reshape(lead) for i, name in enumerate(BUTTONS)}
        out["camera"] = host[:, 20:22].view(np.float64).reshape(*lead, 2)
        return out

    def from_env_device(self, buttons, camera):
        """MineRL env actions on the device -- buttons int64 (n, 20) in `BUTTONS` order, camera float64 (n, 2) degrees -> (joint action
        dict of int64 (n, 1) device tensors, is-null bool (n,)) == from_factored(env2policy(.)) + the null-action test of agent.py:176-180."""
        from . import ops
        t = self._device_tables(buttons.device)
        out = ops.codec_from_env(buttons.to(torch.int64).contiguous(), camera.to(torch.float64).contiguous(), t["thr"], self.n_bins, t["strides"],
                                 self.inventory_idx)
        return dict(buttons=out[:, 0:1], camera=out[:, 1:2]), out[:, 2] != 0

    def policy2env(self, factored):
        """lib/actions.py:154-169."""
        out = {name: factored["buttons"][..., i] for i, name in enumerate(BUTTONS)}
        out["camera"] = self.undiscretize_camera(factored["camera"])
        return out

    def env2policy(self, env_action):
        """lib/actions.py:171-178."""
        nbatch = np.asarray(env_action["camera"]).shape[0]
        dummy = np.zeros((nbatch,))
        return dict(camera=self.discretize_camera(np.asarray(env_action["camera"])),
                    buttons=np.stack([env_action.get(k, dummy) for k in BUTTONS], axis=-1))


# ---------------------------------------------------------------------------------------------------------------------
# frame ingest
# ---------------------------------------------------------------------------------------------------------------------
def _linear_tables(dst: int, src: int):
    """Source index + 11-bit fixed-point weight pairs of OpenCV's 8-bit INTER_LINEAR resize (resize.cpp: fx = (dx+0.5)*scale-0.5,
    cvFloor, clamping at both ends, weights = cvRound(w * 2048) as int16)."""
    scale = src / dst  # double, like resize.cpp's inv_scale_x; fx itself is computed in float there
    idx = np.zeros(dst, dtype=np.int32)
    w = np.zeros((dst, 2), dtype=np.int16)
    for d in range(dst):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        f = np.float32(f - np.float32(s))
        if s < 0:
            s, f = 0, 0.0
        if s >= src - 1:
            s, f = src - 1, 0.0
        idx[d] = s
        w[d, 0], w[d, 1] = int(np.rint((1.0 - f) * 2048)), int(np.rint(f * 2048))
    return idx, w


_TABLE_CACHE = {}


def resize_frames(frames: torch.Tensor, size=AGENT_RESOLUTION, bgr_to_rgb: bool = False) -> torch.Tensor:
    """uint8 CUDA frames [F, Hs, Ws, C] -> [F, size[1], size[0], C], bit-exact with cv2.resize(frame, size, INTER_LINEAR);
    bgr_to_rgb also applies cv2.cvtColor(frame, COLOR_BGR2RGB) (data_loader.py:116) in the same pass."""
    if not frames.is_cuda or frames.dtype != torch.uint8:
        raise nat.NativeError("resize_frames needs a uint8 CUDA tensor (no CPU fallback)")
    frames = frames.contiguous()
    F_, Hs, Ws, C = frames.shape
    Wd, Hd = size
    if Hs < Hd or Ws < Wd:
        # OpenCV takes a different code path when it UPSCALES (measured: +-1 differences against this formula); the
        # reference only ever shrinks 640x360 / 1280x720 frames to 128x128, so upscaling is refused rather than approximated
        raise NotImplementedError("resize_frames is bit-exact with cv2 for downscaling only")
    if Hs == 2 * Hd and Ws == 2 * Wd:
        # OpenCV silently switches INTER_LINEAR to INTER_AREA when both scale factors are exactly 2 (resize.cpp), which this kernel does
        # not implement; the reference never hits it (640x360 / 1280x720 -> 128x128)
        raise NotImplementedError("resize_frames: an exact 2x downscale takes OpenCV's INTER_AREA path, which is not implemented")
    key = (Hs, Ws, Hd, Wd, frames.device)
    if key not in _TABLE_CACHE:
        xi, xw = _linear_tables(Wd, Ws)
        yi, yw = _linear_tables(Hd, Hs)
        _TABLE_CACHE[key] = tuple(torch.from_numpy(a).to(frames.device) for a in (xi, xw, yi, yw))
    xi, xw, yi, yw = _TABLE_CACHE[key]
    out = torch.empty((F_, Hd, Wd, C), dtype=torch.uint8, device=frames.device)
    nat.check(nat.lib().vpt_resize_bilinear_u8(frames.data_ptr(), out.data_ptr(), xi.data_ptr(), xw.data_ptr(), yi.data_ptr(), yw.data_ptr(),
                                               F_, Hs, Ws, Hd, Wd, C, int(bgr_to_rgb), torch.cuda.current_stream().cuda_stream), "vpt_resize_bilinear_u8")
    return out


def composite_cursor(frames: torch.Tensor, cursor: torch.Tensor, alpha: torch.Tensor, xy: torch.Tensor) -> torch.Tensor:
    """In-place cursor overlay of data_loader.py:34-45 on uint8 CUDA frames [F, H, W, 3]: cursor uint8 [ch, cw, 3], alpha float64
    [ch, cw] (= cursor_png[..., 3] / 255.0), xy int32 [F, 2] top-left corner per frame ((-1, -1) = GUI closed, frame untouched)."""
    if not frames.is_cuda or frames.dtype != torch.uint8 or not frames.is_contiguous():
        raise nat.NativeError("composite_cursor needs a contiguous uint8 CUDA tensor (no CPU fallback)")
    F_, H, W, C = frames.shape
    assert C == 3 and cursor.dtype == torch.uint8 and alpha.dtype == torch.float64 and xy.dtype == torch.int32 and tuple(xy.shape) == (F_, 2)
    ch, cw = cursor.shape[:2]
    nat.check(nat.lib().vpt_composite_cursor_u8(frames.data_ptr(), cursor.contiguous().data_ptr(), alpha.contiguous().data_ptr(),
                                                xy.contiguous().data_ptr(), F_, H, W, ch, cw, torch.cuda.current_stream().cuda_stream),
              "vpt_composite_cursor_u8")
    return frames


def ingest_frames(frames_bgr: torch.Tensor, cursor=None, alpha=None, cursor_xy=None, size=AGENT_RESOLUTION) -> torch.Tensor:
    """The BC data loader's per-frame image path on the GPU (data_loader.py:108-118): cursor overlay where the GUI is open ->
    BGR to RGB -> bilinear resize to the agent resolution; uint8 in, uint8 out, bit-exact with the numpy / cv2 code."""
    if cursor is not None:
        frames_bgr = composite_cursor(frames_bgr, cursor, alpha, cursor_xy)
    return resize_frames(frames_bgr, size, bgr_to_rgb=True)


# ---------------------------------------------------------------------------------------------------------------------
# training-time augmentation
# ---------------------------------------------------------------------------------------------------------------------
AUGMENT_PARAMS = ("rotate", "scale", "shear", "translate_x", "translate_y", "brightness", "contrast", "saturation", "hue")


def _check_range(name, r, lo_min, strict=False):
    lo, hi = (float(v) for v in r)
    if not (np.isfinite(lo) and np.isfinite(hi)) or lo > hi or (lo <= lo_min if strict else lo < lo_min):
        raise ValueError(f"augment_params: {name} must be a finite (lo, hi) with {lo_min} {'<' if strict else '<='} lo <= hi (got {r})")
    return lo, hi


def augment_params(B, T=None, *, generator, rotate=0.0, scale=(1.0, 1.0), shear=0.0, translate=0.0, brightness=(1.0, 1.0),
                   contrast=(1.0, 1.0), saturation=(1.0, 1.0), hue=0.0, per_frame=False) -> torch.Tensor:
    """Uniform augmentation parameters for `augment_frames`, fp32 (B, 9) -- one draw per sequence -- or (B, T, 9) with per_frame=True.
    Columns (`AUGMENT_PARAMS`): rotate and shear in degrees, drawn from [-rotate, rotate] and [-shear, shear]; scale from (lo, hi);
    translate_x and translate_y in pixels, each from [-translate, translate]; brightness, contrast and saturation from their (lo, hi);
    hue from [-hue, hue] (hue <= 0.5).  The defaults are the identity.  Every call draws 9 uniforms per row from `generator` (on its
    device) whatever the ranges, so a seeded generator gives the same parameters for the same B, T and per_frame.

    One draw per sequence is the default because the models read motion from differences between neighbouring frames: both policies
    infer the camera action from frame-to-frame image shifts, and the IDM's conv3d mixes five neighbouring frames.  A warp drawn per
    frame would add shifts and rotations that no action caused, contradicting the action labels; `augment_frames` broadcasts a (B, 9)
    draw over the T frames of each sequence."""
    if int(B) != B or B <= 0:
        raise ValueError(f"augment_params: B must be a positive integer (got {B})")
    if per_frame and (T is None or int(T) != T or T <= 0):
        raise ValueError(f"augment_params: per_frame=True needs a positive integer T (got {T})")
    for name, v, ok in (("rotate", rotate, True), ("shear", shear, float(shear) < 90.0), ("translate", translate, True),
                        ("hue", hue, float(hue) <= 0.5)):
        if not (np.isfinite(float(v)) and float(v) >= 0 and ok):
            raise ValueError(f"augment_params: {name} must be a finite half-width >= 0 (shear < 90 degrees, hue <= 0.5; got {v})")
    ranges = [_check_range("scale", scale, 0.0, strict=True), _check_range("brightness", brightness, 0.0),
              _check_range("contrast", contrast, 0.0), _check_range("saturation", saturation, 0.0)]
    n = int(B) * (int(T) if per_frame else 1)
    u = torch.rand((n, 9), generator=generator, dtype=torch.float64, device=generator.device)
    sym = lambda col, r: (2.0 * u[:, col] - 1.0) * float(r)
    lin = lambda col, lh: lh[0] + (lh[1] - lh[0]) * u[:, col]
    p = torch.stack([sym(0, rotate), lin(1, ranges[0]), sym(2, shear), sym(3, translate), sym(4, translate), lin(5, ranges[1]),
                     lin(6, ranges[2]), lin(7, ranges[3]), sym(8, hue)], dim=1).to(torch.float32)
    return p.reshape(int(B), int(T), 9) if per_frame else p


def augment_matrices(params, H, W) -> np.ndarray:
    """float64 (N, 2, 3) inverse affine maps (output pixel -> source point) of `augment_frames` for (N, 9) parameters, about the frame
    centre c = ((W - 1) / 2, (H - 1) / 2), pixel centres at integer coordinates, x right and y down.  The forward map is
        out = c + t + s R(rotate) Sh(shear) (src - c),   R = [[cos, -sin], [sin, cos]],  Sh = [[1, tan], [0, 1]],  t = (tx, ty),
    so a positive rotate turns the content clockwise on screen; the inverse is src = c + L^-1 (out - c - t) with L = s R Sh."""
    p = np.asarray(params, dtype=np.float64).reshape(-1, 9)
    th, s, ph = np.deg2rad(p[:, 0]), p[:, 1], np.deg2rad(p[:, 2])
    cos, sin, tan = np.cos(th), np.sin(th), np.tan(ph)
    # L^-1 = (1/s) Sh^-1 R^T = (1/s) [[cos + tan sin, sin - tan cos], [-sin, cos]]
    li = np.stack([np.stack([cos + tan * sin, sin - tan * cos], -1), np.stack([-sin, cos], -1)], 1) / s[:, None, None]
    c = np.array([(W - 1) / 2.0, (H - 1) / 2.0])
    ct = c[None] + p[:, 3:5]
    off = c[None] - np.einsum("nij,nj->ni", li, ct)
    return np.concatenate([li, off[:, :, None]], axis=2)


def augment_frames(frames: torch.Tensor, params: torch.Tensor, out_dtype=torch.uint8) -> torch.Tensor:
    """Affine and colour jitter of uint8 CUDA frames (N, H, W, 3) or (B, T, H, W, 3) in one kernel (`vpt_augment_frames`): per frame an
    inverse-mapped bilinear warp with zero fill, then brightness, contrast (about the frame's mean grey), saturation and hue, with
    torchvision's `adjust_*` formulas (include/vpt_b200.h states the arithmetic).  `params` (`augment_params`) holds one row per frame,
    (N, 9) or (B, T, 9), or for (B, T, ...) frames (B, 9), one row per sequence broadcast over T.  The output has the frames' shape, uint8
    (rounded to nearest even) or float32 on the uint8 scale (unrounded), which the forward and the trainers take as they are.  The
    inverse matrices are built on the host in float64 (`augment_matrices`) and rounded to fp32; params on the GPU are copied to the host
    first.  Identity parameters return the frames bit for bit.  The output depends on each frame's own bytes and parameters only."""
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
        raise TypeError(f"augment_frames: frames must be a uint8 tensor (got {getattr(frames, 'dtype', type(frames))})")
    if frames.dim() not in (4, 5) or frames.shape[-1] != 3 or frames.numel() == 0:
        raise ValueError(f"augment_frames: frames must be non-empty (N, H, W, 3) or (B, T, H, W, 3) (got {tuple(frames.shape)})")
    if out_dtype not in (torch.uint8, torch.float32):
        raise TypeError(f"augment_frames: out_dtype must be torch.uint8 or torch.float32 (got {out_dtype})")
    rows = augment_rows(params, tuple(frames.shape))
    if not frames.is_cuda:
        raise nat.NativeError("augment_frames needs a CUDA tensor (no CPU fallback)")
    from . import ops
    n, H, W = rows.shape[0], frames.shape[-3], frames.shape[-2]
    frames = frames.contiguous()
    out = torch.empty(frames.shape, dtype=out_dtype, device=frames.device)
    ops.augment(frames.view(n, H, W, 3), torch.from_numpy(rows).to(frames.device), out.view(n, H, W, 3))
    return out


def augment_rows(params, frames_shape) -> np.ndarray:
    """The kernel's per-frame parameters, fp32 (N, 10) = (inverse matrix (2, 3) row-major, brightness, contrast, saturation, hue), for
    `augment_frames` params and frames of shape `frames_shape`; raises ValueError / TypeError on parameters it refuses."""
    if not isinstance(params, torch.Tensor) or not params.dtype.is_floating_point:
        raise TypeError(f"augment_frames: params must be a floating tensor (got {getattr(params, 'dtype', type(params))})")
    lead, (H, W) = tuple(frames_shape[:-3]), tuple(frames_shape[-3:-1])
    n = int(np.prod(lead))
    shapes = [lead + (9,)] + ([(lead[0], 9)] if len(lead) == 2 else [])
    if tuple(params.shape) not in shapes:
        raise ValueError(f"augment_frames: params must be {' or '.join(str(s) for s in shapes)} for frames {tuple(frames_shape)} "
                         f"(got {tuple(params.shape)})")
    p = params.detach().to("cpu", torch.float64).reshape(-1, 9).numpy()
    if p.shape[0] != n:
        p = np.repeat(p, lead[1], axis=0)
    if not np.isfinite(p).all():
        raise ValueError("augment_frames: params must be finite")
    if (p[:, 1] <= 0).any():
        raise ValueError("augment_frames: scale must be > 0")
    if (np.abs(p[:, 2]) >= 90).any():
        raise ValueError("augment_frames: shear must lie in (-90, 90) degrees")
    if (p[:, 5:8] < 0).any():
        raise ValueError("augment_frames: brightness, contrast and saturation must be >= 0")
    if (np.abs(p[:, 8]) > 0.5).any():
        raise ValueError("augment_frames: |hue| must be <= 0.5")
    with np.errstate(over="ignore"):
        A = augment_matrices(p, H, W).astype(np.float32)
    if not np.isfinite(A).all():
        raise ValueError("augment_frames: params give an inverse matrix that is not finite in fp32")
    return np.ascontiguousarray(np.concatenate([A.reshape(n, 6), p[:, 5:9].astype(np.float32)], axis=1))


# ---------------------------------------------------------------------------------------------------------------------
# MineRLAgent
# ---------------------------------------------------------------------------------------------------------------------
class MineRLAgent:
    """agent.py:106-206 without the MineRL / gym dependency: `env` is accepted for signature compatibility and only used to
    check the action-space key set when it exposes one (agent.py:84-97)."""

    def __init__(self, env=None, device=None, policy_kwargs=None, pi_head_kwargs=None, graphed=True):
        from . import PI_HEAD_KWARGS, POLICY_KWARGS_2X

        if env is not None and hasattr(getattr(env, "action_space", None), "spaces"):
            names = set(env.action_space.spaces.keys())
            expected = set(BUTTONS) | {"camera", "ESC", "pickItem", "swapHands"}
            if names != expected:
                raise ValueError(f"MineRL action space does match. Expected actions {expected}")
        self.device = torch.device(device or "cuda")
        self.codec = ActionCodec(**ACTION_TRANSFORMER_KWARGS)
        self.policy = _policy.MinecraftAgentPolicy(action_space=minecraft_action_space(), policy_kwargs=policy_kwargs or POLICY_KWARGS_2X,
                                                   pi_head_kwargs=pi_head_kwargs or PI_HEAD_KWARGS).to(self.device)
        self._graphed = graphed
        self._step = None
        self.hidden_state = self.policy.initial_state(1)
        self._dummy_first = torch.zeros((1,), dtype=torch.bool, device=self.device)

    def load_weights(self, path):
        """agent.py:132-135."""
        from .checkpoint import load_weights
        load_weights(self.policy, path, map_location=self.device)
        self._step = None  # a captured rollout graph belongs to the old weights (GraphedAct re-checks too)
        self.reset()

    def reset(self):
        """agent.py:137-139."""
        self.hidden_state = self.policy.initial_state(1)

    def _env_obs_to_agent(self, minerl_obs):
        """agent.py:141-149: HxWx3 uint8 pov -> {"img": (1,128,128,3) uint8 on the device} (resize on the GPU)."""
        pov = torch.from_numpy(np.ascontiguousarray(minerl_obs["pov"])).to(self.device)
        return {"img": resize_frames(pov[None], AGENT_RESOLUTION)}

    def _agent_action_to_env(self, agent_action):
        """agent.py:151-164.  Device tensors (what `act` returns) are decoded on the GPU: one small device-to-host copy per step."""
        if all(isinstance(v, torch.Tensor) and v.is_cuda for v in agent_action.values()):
            return self.codec.to_env_device(agent_action)
        action = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in agent_action.items()}
        return self.codec.policy2env(self.codec.to_factored(action))

    def _env_action_to_agent(self, minerl_action_transformed, to_torch=False, check_if_null=False):
        """agent.py:166-188."""
        a = self.codec.env2policy(minerl_action_transformed)
        if check_if_null and np.all(a["buttons"] == 0) and np.all(a["camera"] == self.codec.null_bin):
            return None
        if a["camera"].ndim == 1:
            a = {k: v[None] for k, v in a.items()}
        action = self.codec.from_factored(a)
        if to_torch:
            action = {k: torch.from_numpy(v).to(self.device) for k, v in action.items()}
        return action

    def get_action(self, minerl_obs):
        """agent.py:190-206."""
        agent_input = self._env_obs_to_agent(minerl_obs)
        if self._graphed and self._step is None:
            self._step = self.policy.make_graphed_act(1)
        act = self._step if self._graphed else self.policy.act
        agent_action, self.hidden_state, _ = act(agent_input, self._dummy_first, self.hidden_state, stochastic=True)
        return self._agent_action_to_env(agent_action)


# ---------------------------------------------------------------------------------------------------------------------
# IDMAgent
# ---------------------------------------------------------------------------------------------------------------------
class IDMAgent:
    """inverse_dynamics_model.py:20-95 without the gym / cv2 dependency: the inverse dynamics model labelling video frames with
    actions.  The IDM's action space is already factored (IDMActionMapping is the identity, lib/action_mapping.py:102-108), so the
    env action is `ActionCodec.policy2env` of the arg-max heads."""

    def __init__(self, idm_net_kwargs, pi_head_kwargs, device=None):
        from .types import idm_action_space

        self.device = torch.device(device or "cuda")
        self.codec = ActionCodec(**ACTION_TRANSFORMER_KWARGS)
        self.policy = _policy.InverseActionPolicy(idm_action_space(), pi_head_kwargs, idm_net_kwargs).to(self.device)
        self.hidden_state = self.policy.initial_state(1)

    def load_weights(self, path):
        """inverse_dynamics_model.py:45-48."""
        from .checkpoint import load_weights
        load_weights(self.policy, path, map_location=self.device)
        self.reset()

    def reset(self):
        """inverse_dynamics_model.py:50-52."""
        self.hidden_state = self.policy.initial_state(1)

    def _video_obs_to_agent(self, video_frames):
        """inverse_dynamics_model.py:54-59: (N, H, W, 3) uint8 frames -> {"img": (1, N, 128, 128, 3)} on the device (GPU resize)."""
        frames = video_frames if isinstance(video_frames, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(video_frames))
        frames = frames.to(self.device)
        if tuple(frames.shape[1:3]) != (AGENT_RESOLUTION[1], AGENT_RESOLUTION[0]):
            frames = resize_frames(frames, AGENT_RESOLUTION)
        return {"img": frames[None]}

    def _agent_action_to_env(self, agent_action):
        """inverse_dynamics_model.py:61-73."""
        action = {k: v.cpu().numpy() for k, v in agent_action.items()}
        return self.codec.policy2env(action)

    def predict_actions(self, video_frames):
        """inverse_dynamics_model.py:75-95: deterministic action labels for a clip; every head has shape (1, N, ...)."""
        agent_input = self._video_obs_to_agent(video_frames)
        n = agent_input["img"].shape[1]
        dummy_first = torch.zeros((1, n), dtype=torch.bool, device=self.device)  # the unmasked IDM attention ignores `first`
        predicted, self.hidden_state, _ = self.policy.predict(agent_input, first=dummy_first, state_in=self.hidden_state, deterministic=True)
        return self._agent_action_to_env(predicted)
