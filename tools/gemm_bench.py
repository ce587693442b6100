"""Micro-benchmarks of the tensor-core GEMM through the C ABI test hook (CUDA-event timed)."""
import ctypes as C, os, sys, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neuralrecon-w_b200"))
import torch
from nrw import _lib
ap = argparse.ArgumentParser()
ap.add_argument("--one", default="")
a = ap.parse_args()
L = _lib.lib()
dev = "cuda"
def run(M, N, K, planes, act, mn=0, ks=1, iters=6, bias=True):
    if mn:
        A = torch.randn(K, M, device=dev); B = torch.randn(K, N, device=dev) / 30
    else:
        A = torch.randn(M, K, device=dev); B = torch.randn(N, K, device=dev) / 30
    bi = torch.zeros(N, device=dev) if bias else None
    D = torch.zeros(M, N, device=dev)
    scratch = torch.empty(L.nrw_gemm_test_scratch_bytes(M, N, K) + 1024, dtype=torch.uint8, device=dev)
    sp = (scratch.data_ptr() + 1023) // 1024 * 1024
    ts = []
    for it in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(L.nrw_gemm_test(0, planes, mn, ks, M, N, K, _lib.ptr(A), _lib.ptr(B), _lib.ptr(bi), act, _lib.ptr(D), C.c_void_p(sp), _lib.stream_ptr()), "gemm")
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[len(ts)//2]
    nprod = {1:1,2:3,3:6}[planes]
    print(f"M={M} N={N} K={K} planes={planes} act={act} mn={mn} ks={ks}: {ms*1e3:8.1f} us  alg {2*M*N*K/ms/1e9:7.1f} TF  mma {2*M*N*K*nprod/ms/1e9:7.1f} TF")
if a.one:
    M,N,K,p,act,mn,ks = [int(x) for x in a.one.split(",")]
    run(M,N,K,p,act,mn,ks,iters=2)
else:
    for planes in (1,2,3):
        for act in (0,1):
            run(32768, 512, 512, planes, act)
    run(32768, 512, 512, 2, 0, bias=False)
    run(32768, 128, 512, 2, 0)
    run(32768, 512, 64, 2, 1)
    run(131072, 512, 512, 2, 1)
    run(512, 512, 32768, 2, 0, mn=1, ks=18)
    run(512, 512, 32768, 2, 0, mn=1, ks=1)
    run(512, 512, 32768, 1, 0, mn=1, ks=18)
