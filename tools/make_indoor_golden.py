"""Generate tests/golden/indoor_checks.npz from the UNMODIFIED reference (needs the reference tree; CPU only).

Run:  python tools/make_indoor_golden.py
The reference's own NeuconWRenderer + NeuconWLoss + backward, with the background NeRF built as the indoor
configuration builds it (config/train_indoor.yaml: ENCODE_A_BG False -> NeRF(encode_appearance=False); SDF
inside_outside True; 8 + 16 samples in 2 steps, 8 outside samples), no perturbation, on oracle.synth parameters.
Stores every output, the loss, and the gradients (whole up to 2048 elements, else a seeded sample of 1024 elements and
the tensor's max magnitude), plus the no-appearance NeRF's state_dict names and shapes.
"""
import json
import os
import sys
import warnings
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from oracle import make_golden, ref_import, synth  # noqa: E402
from util_indoor import FULL_GRAD_NUMEL, GOLDEN, N_RAYS, RAY_SEED, grad_sample_index, indoor_cfg, indoor_params  # noqa: E402


def main():
    if not ref_import.available():
        print("reference tree not available; cannot regenerate golden vectors", file=sys.stderr)
        sys.exit(1)
    ref = ref_import.load()
    P = indoor_params(seed=0)
    cfg = indoor_cfg(**synth.BRANDENBURG)
    batch = synth.make_rays(N_RAYS, cfg, seed=RAY_SEED)
    full = synth.make_params(seed=0)     # build_reference loads an appearance NeRF; it is replaced below
    with mock.patch.dict(make_golden.SDF_CONFIG, inside_outside=True):
        m = make_golden.build_reference(cfg, full)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        nerf = ref.NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4],
                        encode_appearance=False, in_channels_a=cfg.n_a, in_channels_dir=27, use_viewdirs=True)
    nerf.load_state_dict({k[len("nerf."):]: v for k, v in P.items() if k.startswith("nerf.")}, strict=True)
    m["renderer"].nerf = nerf
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        res = m["renderer"].render(batch["rays"], batch["ts"], batch["label"], perturb_overwrite=0,
                                   background_rgb=torch.zeros([1, 3]), cos_anneal_ratio=cfg.cos_anneal_ratio)
        loss = sum(m["loss"](res, batch["rgbs"]).values())
        loss.backward()
    arrays = {f"out.{k}": v.detach().numpy() for k, v in res.items()}
    arrays["loss"] = loss.detach().numpy()
    for pre, mod in (("neuconw.", m["neuconw"]), ("nerf.", nerf), ("embedding_a.", m["emb"])):
        for k, p in mod.named_parameters():
            name, g = pre + k, (p.grad if p.grad is not None else torch.zeros_like(p)).detach()
            if g.numel() <= FULL_GRAD_NUMEL:
                arrays["g." + name] = g.numpy()
            else:
                arrays["gs." + name] = g.reshape(-1)[grad_sample_index(name, g.numel())].numpy()
                arrays["gmax." + name] = g.abs().max().numpy()
    arrays["nerf_state_dict_shapes"] = np.array(json.dumps({k: list(v.shape) for k, v in nerf.state_dict().items()},
                                                           sort_keys=True))
    np.savez_compressed(GOLDEN, **arrays)
    print(f"wrote {GOLDEN}: loss={float(arrays["loss"]):.6f} {os.path.getsize(GOLDEN) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()
