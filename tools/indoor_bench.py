"""Training-step time of TrainSystem at the indoor configuration's sample counts (config/train_indoor.yaml: 8 + 16 samples
in 2 steps, 8 outside samples), background NeRF without (encode_a_bg False) and with its appearance head.

Both arms live in one process and alternate: every round times `--steps` steps of each arm with CUDA events around
synchronised work, after `--warmup` steps of each.  Reports the median and spread of the per-round mean step time per arm
and their ratio, with the card's name and power limit from a read-only nvidia-smi query.  One JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from nrw.synthetic import make_ray_batch  # noqa: E402
from nrw.train import TrainSystem  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--precision", default="mixed", choices=["bf16x3", "mixed", "bf16", "bf16x6"])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("indoor_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    arms = {}
    for enc in (False, True):
        arms[enc] = TrainSystem(dev, n_samples=8, n_importance=16, up_sample_steps=2, n_outside=8, precision=a.precision,
                                batch_size=a.rays, encode_a_bg=enc, inside_outside=True)
    batch = make_ray_batch(a.rays, seed=1, device=dev)
    for s in arms.values():
        for _ in range(a.warmup):
            s.training_step(batch)
    torch.cuda.synchronize()
    ms = {enc: [] for enc in arms}
    for _ in range(a.rounds):
        for enc, s in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                s.training_step(batch)
            e1.record()
            torch.cuda.synchronize()
            ms[enc].append(e0.elapsed_time(e1) / a.steps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()
    stat = lambda v: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
    res = {"gpu": gpu, "rays": a.rays, "precision": a.precision, "S": 24, "T": 32, "rounds": a.rounds,
           "steps_per_round": a.steps, "encode_a_bg_false": stat(ms[False]), "encode_a_bg_true": stat(ms[True]),
           "ratio_false_over_true": float(np.median(ms[False]) / np.median(ms[True])),
           "slots": {str(enc): list(s.renderer.engine.slots) for enc, s in arms.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
