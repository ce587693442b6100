"""GPU: parity at BASELINE's FULL C2 size against the UNMODIFIED reference itself.

The reference's Python sources travel to the GPU box as the verbatim copy oracle/_ref (oracle/fetch_ref.py), so the real
`NeuconWRenderer.render` + `NeuconWLoss` + `backward` can run there on CUDA (stock torch fp32, TF32 off) on the whole
8192-ray x 128-sample batch of config C2 - no restatement in between.  The reference's autograd graph of all 8192 rays does not fit
an 80 GB GPU, so both sides take the batch as four 2048-ray micro-batches and accumulate the parameter gradient over them, as a
training run on such a GPU would.  Compared with the nrw CUDA path in the headline `mixed` precision on the same rays, same
weights, deterministic strata:

  * every per-ray / per-sample output of the 16-key dict within 1e-4 of its range on all rays whose importance samples fell
    into the same bins (inverse-cdf sampling is discontinuous in the SDF: the number of rays with a flipped bin is reported,
    bounded at 1 %, and those rays are excluded from the element-wise comparison);
    `mask_error` = BCE(clip(weights_sum, 1e-3, 1 - 1e-3), mask) (renderer.py:873-875) is the one ill-conditioned key: its
    derivative in weights_sum reaches 1000 at the clip bounds, so it is held to 1e-3 while weights_sum itself is held to 1e-4;
  * the loss and the eikonal term of every micro-batch within 1e-3 (they average over its rays, flipped ones included);
  * the parameter gradient: cosine >= 0.9999 with the reference's autograd gradient (one-product backward GEMMs and flipped
    rays included), norm ratio within 0.5 %."""
import gc
import json
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import ref_import, synth
from util_nrw import build_system, cuda_train_step, rel_err

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_import.available(), reason="no reference copy (oracle/_ref) on this box")]

PER_RAY = ("color", "color_sphere", "color_bg", "cdf_fine", "gradients", "mask_error", "weights", "weights_sum", "weights_max",
           "inside_sphere", "depth")


MICRO = 2048      # rays per micro-batch: the reference's fp32 autograd graph of all 8192 rays (second-order SDF chain) exceeds 80 GB


def test_full_c2_batch_vs_unmodified_reference_on_gpu():
    from oracle.make_golden import build_reference

    cfg = synth.PathConfig(**synth.BRANDENBURG)                       # C2 counts: 64 + 64, k = 4, 4 outside
    R = 8192
    P = synth.make_params(seed=0)
    batch = synth.make_rays(R, cfg, seed=17)
    parts = [{k: v[i:i + MICRO] for k, v in batch.items()} for i in range(0, R, MICRO)]
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False
    # ---- the unmodified reference on this GPU: the batch as micro-batches, gradients accumulated in .grad ----
    m = build_reference(cfg, P)
    for k in ("neuconw", "nerf", "emb"):
        m[k].to(dev)
    outs_r, z_r, loss_r, gerr_r = [], [], [], []
    for part in parts:
        b = {k: v.to(dev) for k, v in part.items()}
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res_r = m["renderer"].render(b["rays"], b["ts"], b["label"], perturb_overwrite=0,
                                         background_rgb=torch.zeros([1, 3], device=dev), cos_anneal_ratio=cfg.cos_anneal_ratio)
            loss_d = m["loss"](res_r, b["rgbs"])
            loss = sum(loss_d.values())
            loss.backward()
        outs_r.append({k: v.detach().cpu() for k, v in res_r.items()})
        loss_r.append(float(loss.detach()))
        gerr_r.append(float(res_r["gradient_error"].detach()))
        del res_r, loss_d, loss
        # the reference's sampler once more for its z_vals (deterministic: perturb = 0)
        o = ((b["rays"][:, 0:3] - m["renderer"].origin).float() / cfg.radius).float()       # render()'s own normalisation (:813-818)
        with torch.no_grad():
            _, z, _, _ = m["renderer"].sparse_sampler(o, b["rays"][:, 3:6], (b["rays"][:, 6:7] / cfg.radius).float(),
                                                      (b["rays"][:, 7:8] / cfg.radius).float(), 0)
        z_r.append(z.cpu())
        del b, o, z
        gc.collect()
        torch.cuda.empty_cache()
    out_r = {k: torch.cat([o[k] for o in outs_r]) for k in PER_RAY}
    z_r = torch.cat(z_r)
    grads_r = {}
    for pre, mod in (("neuconw.", m["neuconw"]), ("nerf.", m["nerf"])):
        for k, p in mod.named_parameters():
            grads_r[pre + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).detach().cpu()
    del m, outs_r
    gc.collect()
    torch.cuda.empty_cache()
    # ---- nrw, headline precision, the same micro-batches ----
    s = build_system(P, cfg, device=dev, precision="mixed", backend=0)
    outs_c, z_c, loss_c, gerr_c, grads_c = [], [], [], [], {}
    for part in parts:
        o_c, l_c, g_c = cuda_train_step(s, cfg, part, perturb_overwrite=0)
        outs_c.append(o_c)
        loss_c.append(float(l_c))
        gerr_c.append(float(o_c["gradient_error"]))
        z_c.append(s["renderer"].last_extras["z_vals"].cpu())
        for k, g in g_c.items():
            grads_c[k] = grads_c[k] + g if k in grads_c else g
    out_c = {k: torch.cat([o[k] for o in outs_c]) for k in PER_RAY}
    z_c = torch.cat(z_c)
    assert z_c.shape == (R, 128) and out_c["weights"].shape == (R, 132)
    same = ((z_c - z_r).abs().max(dim=1).values <= 2e-5 * float(z_r.abs().max())).numpy()
    flipped = int((~same).sum())
    errs = {}
    for k in PER_RAY:
        a, r = out_c[k].numpy()[same], out_r[k].numpy()[same]
        errs[k] = rel_err(a, r)
    dot = nn = rr = 0.0
    for k, g in grads_r.items():
        gc_ = grads_c[k].double().reshape(-1)
        gr_ = g.double().reshape(-1)
        dot += float((gc_ * gr_).sum()); nn += float((gc_ * gc_).sum()); rr += float((gr_ * gr_).sum())
    cos, ratio = dot / (nn ** 0.5 * rr ** 0.5), (nn / rr) ** 0.5
    report = {"rays": R, "micro_batch_rays": MICRO, "samples": 128, "rays_with_flipped_bins": flipped,
              "output_rel_err": {k: float(f"{v:.3g}") for k, v in errs.items()},
              "loss": [loss_c, loss_r], "gradient_error": [gerr_c, gerr_r], "grad_cosine": cos, "grad_norm_ratio": ratio}
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(report, open(os.path.join(ROOT, "gpurun_out", "fullsize_vs_reference.json"), "w"), indent=1)
    print("[parity] full C2 batch vs the unmodified reference on this GPU:", json.dumps(report))
    assert flipped <= R // 100, flipped
    for k, e in errs.items():
        assert e < (1e-3 if k == "mask_error" else 1e-4), (k, e)
    assert np.array_equal(out_c["inside_sphere"].numpy()[same], out_r["inside_sphere"].numpy()[same])
    for lc, lr, gc_, gr_ in zip(loss_c, loss_r, gerr_c, gerr_r):
        assert abs(lc - lr) < 1e-3 * abs(lr)
        assert abs(gc_ - gr_) < 1e-3 * abs(gr_)
    assert cos >= 0.9999 and abs(ratio - 1.0) < 5e-3, (cos, ratio)
