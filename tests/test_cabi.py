"""CPU: the C-ABI library builds for sm_90a, loads without a GPU and exports every symbol include/vpt_b200.h declares."""
import ctypes
import os
import re

import vpt_b200
from video_pre_training_b200 import _native as nat


def _declared():
    src = open(nat.HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vpt_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_bound_and_exported():
    names = _declared()
    assert len(names) >= 15
    assert set(names) == set(nat.SIGNATURES), set(names) ^ set(nat.SIGNATURES)
    nat.build()
    l = ctypes.CDLL(nat.LIB_PATH)
    for n in names:
        assert hasattr(l, n), f"{n} declared in include/vpt_b200.h but not exported"
    assert l.vpt_abi_version() == 3


def test_library_is_sm90a_wgmma_tma():
    """SASS evidence that the hot kernels are the Hopper-native path (HGMMA = wgmma.mma_async, UTMALDG = TMA, SYNCS = mbarrier)."""
    import shutil
    import subprocess

    nat.build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", nat.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnem in ("HGMMA", "UTMALDG", "SYNCS"):
        assert mnem in sass, mnem


def test_gemm_args_struct_layout_matches_header():
    """ctypes mirror of struct vpt_gemm_args: field order must follow the header."""
    src = open(nat.HEADER).read()
    body = src[src.index("typedef struct vpt_gemm_args {"):src.index("} vpt_gemm_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split("{", 1)[1].split(";"):
        decl = decl.strip()
        if not decl:
            continue
        names = decl.replace("*", " ").split()
        fields += [re.sub(r"\[\d+\]", "", n.strip(",")) for n in decl.replace("*", " ").replace(",", " ").split()[(2 if names[0] == "const" else 1):]]
    assert fields == [f[0] for f in nat.GemmArgs._fields_], (fields, [f[0] for f in nat.GemmArgs._fields_])


def test_no_cpu_fallback():
    import pytest
    import torch

    kw = vpt_b200.policy_kwargs("1x", img_shape=[32, 32, 3], hidsize=256, attention_heads=2, timesteps=8,
                                attention_memory_size=16, n_recurrence_layers=1)
    pol = vpt_b200.MinecraftAgentPolicy(vpt_b200.minecraft_action_space(), kw, vpt_b200.PI_HEAD_KWARGS)
    img = torch.zeros(1, 1, 32, 32, 3, dtype=torch.uint8)
    with pytest.raises(nat.NativeError):
        pol({"img": img}, torch.zeros(1, 1, dtype=torch.bool), pol.initial_state(1))
