"""Long KV memories on the CPU: tests/golden/long_memory.pt is still what the reference computes (re-derived live where the reference
checkout is present), and `resize_memory` lets 128-frame weights load into a policy with a 1920-frame memory, with the same outputs on a
first chunk (through the oracle)."""
import os
import sys

import pytest
import torch

import refshim
import vpt_b200
import vpt_oracle as O
from common import make_policy, small_kwargs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_long_memory_golden as MLG  # noqa: E402


def _close(a, b, what):
    if isinstance(a, dict):
        assert set(a) == set(b), what
        for k in a:
            _close(a[k], b[k], f"{what}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _close(x, y, f"{what}[{i}]")
    elif isinstance(a, torch.Tensor):
        assert a.shape == b.shape and a.dtype == b.dtype, what
        if a.dtype == torch.bool or not a.dtype.is_floating_point:
            assert torch.equal(a, b), what
        else:
            scale = max(b.abs().max().item(), 1e-12)
            assert (a - b).abs().max().item() <= 1e-5 * scale, what
    else:
        assert a == b, what


def test_fixture_shapes():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "long_memory.pt"), weights_only=False)
    for name, (ams, T, *_) in MLG.CONFIGS.items():
        maxlen = ams - T
        assert fx[name]["policy_kwargs"]["attention_memory_size"] == ams and fx[name]["policy_kwargs"]["timesteps"] == T
        b_nd = [g for n, g in fx[name]["window"]["grads"].items() if n.endswith("orc_block.b_nd")]
        assert b_nd and all(g["shape"] == (10, maxlen) for g in b_nd)
        for m, k, v in fx[name]["forward"]["state"]:
            assert m.shape == (MLG.B, 1, maxlen) and k.shape == (MLG.B, len(MLG.state_rows(maxlen)), 256)
            assert m.any() and not m.all()  # the episode start hid part of row 1's memory


@pytest.mark.skipif(not refshim.available(), reason="needs the reference checkout")
def test_fixture_is_what_the_reference_computes():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "long_memory.pt"), weights_only=False)
    _close(MLG.make_long_memory(), fx, "long_memory")


def test_resize_memory_cuts_and_pads_b_nd():
    _, sd, _ = make_policy(small_kwargs(timesteps=128, attention_memory_size=256), pert=False)
    keys = [k for k in sd if k.endswith("orc_block.b_nd")]
    assert len(keys) == 2
    big = vpt_b200.resize_memory(sd, 1920)
    small = vpt_b200.resize_memory(big, 64)
    for k in keys:
        assert big[k].shape == (10, 1920) and torch.equal(big[k][:, :128], sd[k]) and not big[k][:, 128:].any()
        assert torch.equal(small[k], sd[k][:, :64])
    assert all(big[k] is sd[k] for k in sd if k not in keys)
    assert sd[keys[0]].shape == (10, 128)  # the input is left alone
    with pytest.raises(ValueError):
        vpt_b200.resize_memory(sd, -1)


def test_resize_memory_loads_into_a_longer_memory_with_the_same_first_chunk():
    kw128 = small_kwargs(timesteps=128, attention_memory_size=256)
    kw1920 = small_kwargs(timesteps=128, attention_memory_size=2048)
    _, sd, cfg128 = make_policy(kw128)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw1920, vpt_b200.PI_HEAD_KWARGS)
    with pytest.raises(RuntimeError):
        pol.load_state_dict(sd, strict=False)
    pol.load_state_dict(vpt_b200.resize_memory(sd, 1920))
    sd1920 = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    g = torch.Generator().manual_seed(4)
    img = torch.randint(0, 256, (2, 128, 32, 32, 3), dtype=torch.uint8, generator=g)
    first = torch.zeros(2, 128, dtype=torch.bool)
    cfg1920 = O.Cfg(**kw1920)
    with torch.no_grad():
        (pa, va, _), _ = O.agent_policy_forward(sd, cfg128, img, first, O.initial_state(cfg128, 2))
        (pb, vb, _), _ = O.agent_policy_forward(sd1920, cfg1920, img, first, O.initial_state(cfg1920, 2))
    for k in pa:
        err = ((pb[k] - pa[k]).abs() / pa[k].abs().clamp(min=1e-30)).max().item()
        assert err < 1e-4, (k, err)
    assert ((vb - va).abs() / va.abs().clamp(min=1e-30)).max().item() < 1e-4
