"""Hardware experiment: does a K-major SWIZZLE_128B wgmma descriptor whose start address is advanced by s rows (s*128 B, not
1024-aligned) read rows s.. of the tile correctly, and does it need the base_offset field?  csrc/conv_zp.cuh relies on the answer
(on an H100: correct with base_offset 0 for every shift; setting the field breaks every shift that is not a multiple of 8)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import vpt_b200
from video_pre_training_b200 import _native as nat, ops
l = nat.lib()
g = torch.Generator().manual_seed(0)
M, N, K = 512, 128, 256
A = torch.randn(M, K, generator=g).to(torch.bfloat16)
B = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16)
ref = A.float() @ B.float().T
for s in (0, 1, 2, 3, 5, 8, 9, 16, 37):
    for bo in (0, 1):
        l.vpt_debug_set(s, bo)
        out = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
        ops.gemm(A.cuda(), B.cuda(), out, M, N, K, cluster=1)
        nat.device_check()
        o = out.float().cpu().reshape(M // 128, 128, N)[:, : 128 - s]
        r = ref.reshape(M // 128, 128, N)[:, : 128 - s]
        err = ((o - r).norm() / r.norm()).item()
        print(f"shift {s:3d} base_offset_mode {bo}: rel l2 err of the valid rows {err:.3e}  {'OK' if err < 1e-2 else 'WRONG'}")
l.vpt_debug_set(0, 0)
