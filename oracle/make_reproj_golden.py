"""Recipe: tests/golden/reproj_error.npz, the seeded scene of oracle/trackerr_port.make_scene and what the UNMODIFIED
tools/reproj_error.py computes on it (TEST INFRASTRUCTURE; data only).

    python -m oracle.make_reproj_golden        (needs the reference tree; runs it on the CPU)

Stored: the scene arrays (object arrays flattened to CSR), and the reference's GT index per track, errors per
observation in track order, their mean and the rows of colmap_sfm.ply."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "reproj_error.npz")
SEED = 0


def _csr(arrays, width):
    off = np.zeros(len(arrays) + 1, np.int64)
    off[1:] = np.cumsum([len(a) for a in arrays])
    flat = np.concatenate([np.asarray(a).reshape(-1, width) for a in arrays]) if len(arrays) else np.zeros((0, width))
    return flat, off


def pack(sc):
    out = {k: v for k, v in sc.items() if k not in ("xys", "pids", "track")}
    out["xys"], out["xys_off"] = _csr(sc["xys"], 2)
    out["pids"], _ = _csr(sc["pids"], 1)
    out["track"], out["track_off"] = _csr(sc["track"], 2)
    return out


def unpack(z):
    """the make_scene dict back from the npz"""
    sc = {k: z[k] for k in z.files if not k.startswith("ref_") and k not in ("xys_off", "track_off")}
    xo, to = z["xys_off"], z["track_off"]

    def obj(flat, off, shape):
        a = np.empty(len(off) - 1, dtype=object)
        for i in range(len(off) - 1):
            a[i] = flat[off[i]:off[i + 1]].reshape(shape)
        return a

    sc["xys"] = obj(z["xys"], xo, (-1, 2))
    sc["pids"] = obj(z["pids"].reshape(-1).astype(np.int64), xo, (-1,))
    sc["track"] = obj(z["track"].astype(np.int64), to, (-1, 2))
    for k in ("track_length", "reproj_error", "img_reproj_error"):
        sc[k] = sc[k].item()
    return sc


def reference_rows(sc, workdir):
    """run the unmodified gt_reproject_error on the scene (cwd = workdir) with a GT-index recorder around get_gt_point"""
    import contextlib
    import io

    import torch

    from oracle import trackerr_port as tp

    ref = tp.load_reference()
    gp = tp.write_scene(workdir, sc)
    rec = []
    get = ref.get_gt_point

    def recording(pcd, cam_pose, cam_intrinsic, track_pts2D):
        out = get(pcd, cam_pose, cam_intrinsic, track_pts2D)
        full = torch.cat([pcd, torch.ones(pcd.shape[0], 1)], -1)
        for row in out.reshape(-1, 4):
            rec.append(int(torch.nonzero((full == row).all(1))[0, 0]))
        return out

    ref.get_gt_point = recording
    cwd = os.getcwd()
    os.chdir(workdir)
    try:
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            loss = ref.gt_reproject_error(workdir, gp, np.array(sc["sfm2gt"]), "dense/sparse", sc["track_length"],
                                          sc["reproj_error"], 2, sc["img_reproj_error"])
    finally:
        os.chdir(cwd)
        ref.get_gt_point = get
    errors = np.asarray(ref.plt.plot.call_args[0][1], np.float64)
    return ref, float(loss), np.array(rec, np.int64), errors


def main():
    import tempfile

    import torch

    sys.path[:0] = [ROOT, os.path.join(ROOT, "neuralrecon-w_b200")]
    torch.Tensor.cuda = lambda self, *a, **k: self
    from oracle import trackerr_port as tp

    sc = tp.make_scene(seed=SEED)
    with tempfile.TemporaryDirectory() as d:
        ref, loss, gt_index, errors = reference_rows(sc, d)
        sfm = ref.written["samples/reproject/colmap_sfm.ply"]
    np.savez_compressed(OUT, **pack(sc), ref_loss=loss, ref_gt_index=gt_index, ref_errors=errors, ref_colmap_sfm=sfm)
    print(f"wrote {OUT}: {len(gt_index)} tracks, loss {loss}")


if __name__ == "__main__":
    main()
