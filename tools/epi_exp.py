"""Tuning experiment: time ONE GEMM launch (live CUDA events inside the library) for a forward-layer shaped problem.
Env: NRW_GEMM_TEST_LAYER=1 (layer store pattern)."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neuralrecon-w_b200"))
import torch
from nrw import _lib
L = _lib.lib()
M, N, K, planes, act = [int(x) for x in (sys.argv[1] if len(sys.argv) > 1 else "262144,512,512,2,1").split(",")]
A = torch.randn(M, K, device="cuda"); B = torch.randn(N, K, device="cuda") / 30
bi = torch.zeros(N, device="cuda"); D = torch.zeros(M, N, device="cuda")
scratch = torch.empty(L.nrw_gemm_test_scratch_bytes(M, N, K) + 1024, dtype=torch.uint8, device="cuda")
sp = (scratch.data_ptr() + 1023) // 1024 * 1024
def call():
    _lib.check(L.nrw_gemm_test(0, planes, 0, 1, M, N, K, _lib.ptr(A), _lib.ptr(B), _lib.ptr(bi), act, _lib.ptr(D), C.c_void_p(sp), _lib.stream_ptr()), "gemm")
for _ in range(3): call()
torch.cuda.synchronize()
L.nrw_gemm_timing(1, None)
for _ in range(5): call()
torch.cuda.synchronize()
out = (C.c_double * 5)()
L.nrw_gemm_timing(0, out)
ms = out[0] / out[3]
print(f"LAYER={os.environ.get('NRW_GEMM_TEST_LAYER','0')} M={M} N={N} K={K} P={planes} act={act}: {ms*1e3:.1f} us/launch  mma {out[2]/out[0]/1e9:.0f} TF/s")
