"""Cost of one appearance-code fitting step: colour loss, backward and Adam over the codes of --rays rays at C2's sampling
(64 + 64 samples in 4 steps, 4 outside, no perturbation) on frozen networks, in two arms:

  cache   AppearanceCache(renderer, rays, ts)(codes) (nrw_appearance_forward / _backward on the prepared cache)
  render  renderer.render(rays, ts) + backward with the network parameters frozen (requires_grad False) and the codes a
          leaf: the whole training forward and backward, sampler included

The arms alternate: every round times `--steps` steps of each arm with CUDA events around synchronised work, after
`--warmup` steps of each.  The cache's one-off prepare is timed separately.  Reports the median and spread of the
per-round mean step time per arm and their ratio, with the card's name and power limit from a read-only nvidia-smi query.
One JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from nrw.appearance import AppearanceCache, color_loss  # noqa: E402
from util_nrw import build_system, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--precision", default="mixed", choices=["bf16x3", "mixed", "bf16", "bf16x6"])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("appearance_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    cfg = synth.C2
    s = build_system(synth.make_params(seed=0), cfg, device=dev, precision=a.precision, backend=0)
    r, emb = s["renderer"], s["emb"]
    for m in (s["neuconw"], s["nerf"], emb):
        m.requires_grad_(False)
    batch = {k: v.to(dev) for k, v in synth.make_rays(a.rays, cfg, seed=1).items()}
    rays, ts, rgbs = batch["rays"], batch["ts"], batch["rgbs"]
    codes = emb.weight[ts].detach().clone().requires_grad_(True)
    opt = torch.optim.Adam([codes], lr=1e-3)
    bg = torch.zeros(1, 3, device=dev)

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    cache = AppearanceCache(r, rays, ts, background_rgb=bg)
    e1.record()
    torch.cuda.synchronize()
    prepare_ms = e0.elapsed_time(e1)

    def step_cache():
        opt.zero_grad(set_to_none=True)
        color_loss(cache(codes), rgbs).backward()
        opt.step()

    def step_render():
        opt.zero_grad(set_to_none=True)
        r.embeddings = {"a": lambda t: codes}
        try:
            out = r.render(rays, ts, batch["label"], perturb_overwrite=0, background_rgb=bg)
        finally:
            r.embeddings = {"a": emb}
        color_loss(out["color"], rgbs).backward()
        opt.step()

    arms = {"cache": step_cache, "render": step_render}
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
    res = {"gpu": gpu, "rays": a.rays, "samples_per_ray": cache.S, "n_outside": cache.n_outside, "precision": a.precision,
           "chunk_rows": r.engine.bound[3], "rounds": a.rounds, "steps_per_round": a.steps, "prepare_ms": prepare_ms,
           **{k: stat(v) for k, v in ms.items()},
           "ratio_render_over_cache": float(np.median(ms["render"]) / np.median(ms["cache"]))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
