"""Cost of differentiating a point query: an eikonal loss ((NeuconW.gradient(x).norm(dim=-1) - 1)**2).mean() at --points
random points, forward and backward (the backward recomputes the query's forward, nrw_neuconw_backward), against the
forward alone (the same call under no_grad).

The two arms alternate: every round times `--steps` calls of each arm with CUDA events around synchronised work, after
`--warmup` calls of each.  Reports the median and spread of the per-round mean call time per arm and their ratio, with the
card's name and power limit from a read-only nvidia-smi query.  One JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nrw  # noqa: E402
from nrw.engine import Engine  # noqa: E402
from oracle import synth  # noqa: E402

SDF_CONFIG = dict(d_in=3, d_out=513, d_hidden=512, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1,
                  geometric_init=True, weight_norm=True, inside_outside=False)
COLOR_CONFIG = dict(d_in=9, d_feature=512, mode="idr", d_out=3, d_hidden=256, n_layers=4, head_channels=128,
                    static_head_layers=2, weight_norm=True, multires_view=4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1 << 20)
    ap.add_argument("--precision", default="mixed", choices=["bf16x3", "mixed", "bf16", "bf16x6"])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("query_bwd_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    P = synth.make_params(seed=0)
    neuconw = nrw.NeuconW(SDF_CONFIG, COLOR_CONFIG, dict(init_val=0.3), in_channels_a=48, encode_a=True)
    neuconw.load_state_dict({k[len("neuconw."):]: v for k, v in P.items() if k.startswith("neuconw.")})
    neuconw = neuconw.to(dev)
    eng = Engine(neuconw=neuconw, nerf=None, n_a=48, precision=a.precision)
    g = torch.Generator(device=dev).manual_seed(0)
    x0 = torch.rand(a.points, 3, device=dev, generator=g) * 1.6 - 0.8

    def forward_only():
        with torch.no_grad():
            ((neuconw.gradient(x0.clone()).norm(dim=-1) - 1) ** 2).mean()

    def forward_backward():
        neuconw.zero_grad(set_to_none=True)
        x = x0.clone()
        ((neuconw.gradient(x).norm(dim=-1) - 1) ** 2).mean().backward()

    arms = {"forward": forward_only, "forward_backward": forward_backward}
    for f in arms.values():
        for _ in range(a.warmup):
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / a.steps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()
    stat = lambda v: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
    res = {"gpu": gpu, "points": a.points, "precision": a.precision, "chunk_rows": eng.bound[3], "rounds": a.rounds,
           "steps_per_round": a.steps, **{k: stat(v) for k, v in ms.items()},
           "ratio_forward_backward_over_forward": float(np.median(ms["forward_backward"]) / np.median(ms["forward"]))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
