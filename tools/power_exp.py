"""Is the GEMM power-capped?  Runs ~1.5 s of back-to-back launches of one shape and samples SM clock and board power
through NVML meanwhile."""
import ctypes as C, os, sys, threading, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "neuralrecon-w_b200"))
import torch, pynvml as nv
from nrw import _lib
L = _lib.lib()
M, N, K, planes, act = 262144, 512, 512, int(os.environ.get("P", 2)), 1
A = torch.randn(M, K, device="cuda"); B = torch.randn(N, K, device="cuda") / 30
bi = torch.zeros(N, device="cuda"); D = torch.zeros(M, N, device="cuda")
scratch = torch.empty(L.nrw_gemm_test_scratch_bytes(M, N, K) + 1024, dtype=torch.uint8, device="cuda")
sp = (scratch.data_ptr() + 1023) // 1024 * 1024
def call():
    _lib.check(L.nrw_gemm_test(0, planes, 0, 1, M, N, K, _lib.ptr(A), _lib.ptr(B), _lib.ptr(bi), act, _lib.ptr(D), C.c_void_p(sp), _lib.stream_ptr()), "gemm")
nv.nvmlInit(); h = nv.nvmlDeviceGetHandleByIndex(0)
for _ in range(20): call()
torch.cuda.synchronize()
clk, pw, stop = [], [], threading.Event()
def samp():
    while not stop.is_set():
        clk.append(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)); pw.append(nv.nvmlDeviceGetPowerUsage(h) / 1e3); time.sleep(0.05)
th = threading.Thread(target=samp); th.start()
L.nrw_gemm_timing(1, None)
t0 = time.time()
while time.time() - t0 < 1.5:
    for _ in range(50): call()
    torch.cuda.synchronize()
out = (C.c_double * 5)(); L.nrw_gemm_timing(0, out)
stop.set(); th.join()
clk.sort(); pw.sort()
print(f"LAYER={os.environ.get('NRW_GEMM_TEST_LAYER','0')} P={planes}: {out[0]/out[3]*1e3:.1f} us/launch over {int(out[3])} launches; "
      f"SM clock median {clk[len(clk)//2]} MHz (min {clk[0]}), power median {pw[len(pw)//2]:.0f} W (max {pw[-1]:.0f}), limit {nv.nvmlDeviceGetEnforcedPowerLimit(h)/1e3:.0f} W")
