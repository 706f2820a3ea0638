"""CPU: the host side of the training-time augmentation -- `augment_params` (shapes, ranges, per-sequence draws, reproducibility), the
inverse matrices of `augment_matrices` against a float64 restatement by 3 x 3 matrix inversion, and every call `augment_frames` refuses
raising before any op runs.  tests/test_gpu_augment.py checks the kernel."""
import math

import numpy as np
import pytest
import torch

import vpt_b200  # noqa: F401  (registers the package under its import name)
from video_pre_training_b200 import _native as nat
from video_pre_training_b200 import ops
from video_pre_training_b200.agent import AUGMENT_PARAMS, augment_frames, augment_matrices, augment_params

RANGES = dict(rotate=10.0, scale=(0.9, 1.1), shear=5.0, translate=4.0, brightness=(0.8, 1.2), contrast=(0.7, 1.3), saturation=(0.5, 1.5),
              hue=0.1)


def test_params_shapes_and_per_sequence_default():
    p = augment_params(4, 16, generator=torch.Generator().manual_seed(0), **RANGES)
    assert p.dtype == torch.float32 and tuple(p.shape) == (4, 9) and len(AUGMENT_PARAMS) == 9
    q = augment_params(4, 16, generator=torch.Generator().manual_seed(0), per_frame=True, **RANGES)
    assert q.dtype == torch.float32 and tuple(q.shape) == (4, 16, 9)
    assert tuple(augment_params(3, generator=torch.Generator().manual_seed(0)).shape) == (3, 9)
    with pytest.raises(ValueError, match="per_frame"):
        augment_params(3, generator=torch.Generator(), per_frame=True)


def test_params_defaults_are_identity():
    p = augment_params(64, generator=torch.Generator().manual_seed(1))
    assert torch.equal(p, torch.tensor([0, 1, 0, 0, 0, 1, 1, 1, 0], dtype=torch.float32).expand(64, 9))


def test_params_ranges_and_reproducibility():
    g = torch.Generator().manual_seed(2)
    p = augment_params(4096, generator=g, **RANGES).double()
    col = {n: p[:, i] for i, n in enumerate(AUGMENT_PARAMS)}
    for name, half in (("rotate", 10.0), ("shear", 5.0), ("translate_x", 4.0), ("translate_y", 4.0), ("hue", 0.1)):
        assert col[name].abs().max() <= half and col[name].min() < -0.9 * half and col[name].max() > 0.9 * half, name
        assert abs(col[name].mean().item()) < 0.05 * half, name
    for name, (lo, hi) in (("scale", (0.9, 1.1)), ("brightness", (0.8, 1.2)), ("contrast", (0.7, 1.3)), ("saturation", (0.5, 1.5))):
        assert col[name].min() >= np.float32(lo) and col[name].max() <= np.float32(hi), name
        assert col[name].min() < lo + 0.05 * (hi - lo) and col[name].max() > hi - 0.05 * (hi - lo), name
    # the columns are independent draws
    c = torch.corrcoef(p.T)
    assert (c - torch.eye(9, dtype=c.dtype)).abs().max() < 0.1
    again = augment_params(4096, generator=torch.Generator().manual_seed(2), **RANGES).double()
    assert torch.equal(p, again)
    other = augment_params(4096, generator=torch.Generator().manual_seed(3), **RANGES).double()
    assert not torch.equal(p, other)
    # the same generator state gives the same draw whatever the ranges: 9 uniforms per row are always consumed
    a = augment_params(8, generator=torch.Generator().manual_seed(4), rotate=3.0)
    b = augment_params(8, generator=torch.Generator().manual_seed(4), **RANGES)
    u = (a[:, 0].double() / 3.0 + 1.0) / 2.0
    assert torch.allclose(b[:, 0].double(), (2.0 * u - 1.0) * 10.0, atol=1e-5)


@pytest.mark.parametrize("kw", [dict(rotate=-1.0), dict(rotate=math.inf), dict(shear=90.0), dict(translate=-0.5), dict(hue=0.6),
                                dict(hue=-0.1), dict(scale=(0.0, 1.0)), dict(scale=(1.2, 1.1)), dict(brightness=(-0.1, 1.0)),
                                dict(contrast=(1.0, math.nan)), dict(saturation=(2.0, 1.0))])
def test_params_refuse_bad_ranges(kw):
    with pytest.raises(ValueError):
        augment_params(2, generator=torch.Generator(), **kw)


def _restated(p, H, W):
    """float64: the inverse of the 3 x 3 forward map T(c + t) R Sh S T(-c)."""
    out = []
    for r in np.asarray(p, dtype=np.float64):
        th, s, ph = math.radians(r[0]), r[1], math.radians(r[2])
        c = np.array([(W - 1) / 2.0, (H - 1) / 2.0])
        T = lambda v: np.array([[1, 0, v[0]], [0, 1, v[1]], [0, 0, 1.0]])
        R = np.array([[math.cos(th), -math.sin(th), 0], [math.sin(th), math.cos(th), 0], [0, 0, 1.0]])
        Sh = np.array([[1, math.tan(ph), 0], [0, 1, 0], [0, 0, 1.0]])
        S = np.diag([s, s, 1.0])
        fwd = T(c + r[3:5]) @ R @ Sh @ S @ T(-c)
        out.append(np.linalg.inv(fwd)[:2])
    return np.stack(out)


@pytest.mark.parametrize("H,W", [(128, 128), (96, 160)])
def test_inverse_matrices_match_float64(H, W):
    p = augment_params(256, generator=torch.Generator().manual_seed(5), rotate=30.0, scale=(0.5, 2.0), shear=20.0, translate=20.0).numpy()
    got = augment_matrices(p, H, W)
    assert got.dtype == np.float64 and got.shape == (256, 2, 3)
    ref = _restated(p, H, W)
    assert np.abs(got - ref).max() < 1e-11
    # the forward map of each row sends its inverse's source point back to the output pixel
    ident = augment_matrices(np.array([[0, 1, 0, 0, 0, 1, 1, 1, 0]]), H, W)
    assert np.array_equal(ident[0], np.array([[1.0, 0, 0], [0, 1.0, 0]]))
    shift = augment_matrices(np.array([[0, 1, 0, 3, -2, 1, 1, 1, 0]]), H, W)
    assert np.array_equal(shift[0], np.array([[1.0, 0, -3], [0, 1.0, 2]]))


@pytest.fixture()
def recorder(monkeypatch):
    calls = []
    monkeypatch.setattr(ops, "augment", lambda *a, **k: calls.append(a))
    return calls


def _refused(calls, exc, fn, match):
    with pytest.raises(exc, match=match):
        fn()
    assert calls == []


def _ident(n):
    return torch.tensor([0, 1, 0, 0, 0, 1, 1, 1, 0], dtype=torch.float32).repeat(n, 1)


def test_refusals_raise_before_any_op(recorder):
    f = torch.zeros(4, 8, 8, 3, dtype=torch.uint8)
    seq = torch.zeros(2, 3, 8, 8, 3, dtype=torch.uint8)
    p = _ident(4)
    _refused(recorder, nat.NativeError, lambda: augment_frames(f, p), "CUDA")
    _refused(recorder, nat.NativeError, lambda: augment_frames(seq, _ident(2)), "CUDA")
    _refused(recorder, TypeError, lambda: augment_frames(f.float(), p), "uint8")
    _refused(recorder, TypeError, lambda: augment_frames(f.to(torch.int16), p), "uint8")
    _refused(recorder, ValueError, lambda: augment_frames(torch.zeros(4, 8, 8, 4, dtype=torch.uint8), p), "shape|H, W, 3")
    _refused(recorder, ValueError, lambda: augment_frames(torch.zeros(8, 8, 3, dtype=torch.uint8), p), "H, W, 3")
    _refused(recorder, ValueError, lambda: augment_frames(torch.zeros(0, 8, 8, 3, dtype=torch.uint8), _ident(0)), "non-empty")
    _refused(recorder, TypeError, lambda: augment_frames(f, p, out_dtype=torch.float16), "out_dtype")
    _refused(recorder, TypeError, lambda: augment_frames(f, p.to(torch.int32)), "floating")
    _refused(recorder, ValueError, lambda: augment_frames(f, _ident(3)), "params must be")
    _refused(recorder, ValueError, lambda: augment_frames(f, _ident(4)[:, :8]), "params must be")
    _refused(recorder, ValueError, lambda: augment_frames(seq, _ident(3)), "params must be")
    _refused(recorder, ValueError, lambda: augment_frames(seq, _ident(6)), "params must be")
    for col, val, match in ((0, math.nan, "finite"), (3, math.inf, "finite"), (1, 0.0, "scale"), (1, -1.0, "scale"), (5, -0.1, ">= 0"),
                            (6, -1.0, ">= 0"), (7, -2.0, ">= 0"), (8, 0.51, "hue"), (8, -0.6, "hue"), (2, 90.0, "shear"), (2, -95.0, "shear"),
                            (1, 1e-39, "not finite")):
        bad = p.clone()
        bad[2, col] = val
        _refused(recorder, ValueError, lambda: augment_frames(f, bad), match)
        bad_seq = _ident(2)
        bad_seq[1, col] = val
        _refused(recorder, ValueError, lambda: augment_frames(seq, bad_seq), match)
    # valid per-frame and per-sequence shapes get as far as the device check
    _refused(recorder, nat.NativeError, lambda: augment_frames(seq, _ident(6).view(2, 3, 9)), "CUDA")
    _refused(recorder, nat.NativeError, lambda: augment_frames(seq, _ident(2).double()), "CUDA")
