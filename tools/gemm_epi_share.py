"""Cycle attribution of the tensor-core GEMM over one C2 training step (TcParams::prof, armed through
nrw_debug_gemm_profile): summed over every GEMM launch of the step and every CTA, per consumer warpgroup, the share of
kernel cycles its first warp spent waiting for TMA data, waiting for its turn at the tensor cores and in the epilogue.
usage: python tools/gemm_epi_share.py [precision]      (NRW_LIB_PATH selects an alternate build)"""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "neuralrecon-w_b200"))
import torch
import bench
from nrw import _lib
from nrw.train import TrainSystem
from nrw.synthetic import make_ray_batch

precision = sys.argv[1] if len(sys.argv) > 1 else "mixed"
w = dict(bench.WORKLOADS["C2"]); dev = torch.device("cuda:0")
sysm = TrainSystem(dev, n_samples=w["n_samples"], n_importance=w["n_importance"], up_sample_steps=w["up_sample_steps"],
                   n_outside=w["n_outside"], precision=precision, chunk_rows=262144, batch_size=w["rays"], world_size=1, seed=66)
b = {k: v.to(dev) for k, v in make_ray_batch(w["rays"], seed=1).items()}
for _ in range(2):
    sysm.training_step(b)
L = _lib.lib()
n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
prof = torch.zeros(n_sm * 16, dtype=torch.int64, device=dev)
torch.cuda.synchronize()
L.nrw_debug_gemm_profile(C.c_void_p(prof.data_ptr()))
sysm.training_step(b)
torch.cuda.synchronize()
L.nrw_debug_gemm_profile(None)
s = prof.view(n_sm, 16).double().sum(0).tolist()
kern = s[5]
print(f"{precision}: kernel cycles summed over CTAs {kern:.4g}; producer waiting for a free stage {100 * s[0] / kern:.1f} %")
for wg in range(2):
    o = 8 * wg
    n = s[6 + o] + s[7 + o]
    if n == 0:
        continue
    print(f"  warpgroup {wg}: tiles {s[6 + o]:.0f}  paired dW items {s[7 + o]:.0f}  TMA wait {100 * s[1 + o] / kern:5.1f} %"
          f"  tensor-core turn wait {100 * s[3 + o] / kern:5.1f} %  epilogue {100 * s[4 + o] / kern:5.1f} %"
          f"  epilogue per item {s[4 + o] / n:.0f} cycles")
