"""Generate tests/golden/*.npz from the REFERENCE's own CUDA kernels (oracle/_ref/*.so, built by
`make -C oracle ref REFERENCE=<reference checkout>` from its unmodified sources).  Needs a GPU and oracle/liboracle.so:

    python tests/golden/make_golden.py OUT_DIR          # then copy OUT_DIR/*.npz into tests/golden/
    python tests/golden/make_golden.py OUT_DIR geometry # only roi_align_geometry_sm90a.npz (tests/geometry_cases.py)

Inputs are the seeded cases of tests/cases.py and synthetic.py, so only the reference OUTPUTS are stored.  Outputs of the
full-size configurations are stored as a fixed, seeded sample of positions (roi_align_full_size.npz,
roi_align_bwd_spread.npz) to keep the files small.

The per-case files of the small cases (roi_align_xfrom_<case>, legacy_pool_*, roi_crop, nms) were recorded from the
reference built for sm_100a; the RoIAlign forward of its sm_90a build rounds some outputs 1 ulp apart from them, so an
H100 run must not replace roi_align_xfrom_<case>.npz.  The same RoIAlign outputs of the sm_90a build go to
roi_align_xfrom_sm90a.npz; it and the full-size files were recorded on an H100.  The other kernels' outputs of the sm_90a
build, generated on an H100 from the same inputs, were checked against the stored sm_100a files: the legacy RoIAlign
forward, RoIPool output / argmax / gradient, RoICrop output and grid gradient and every NMS keep list are bit-identical; the
legacy RoIAlign and RoICrop image gradients, which both builds sum with fp32 atomics, differ by at most 3.4e-6 and 1.2e-7,
inside the tests' 1e-5 + 1e-5 |x| tolerance.  So those files stand for both builds.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import gpu_ref as G      # noqa: E402
from oracle import cpu as O          # noqa: E402
from tests import cases              # noqa: E402

SAMPLE = 8192


def _sample(a, seed, nonzero=False):
    """Sorted flat positions of a fixed, seeded sample of `a` (of its non-zero elements if `nonzero`)."""
    pool = np.flatnonzero(a) if nonzero else np.arange(a.size)
    pick = np.random.RandomState(seed).choice(pool.size, min(SAMPLE, pool.size), replace=False)
    return np.sort(pool[pick]).astype(np.int64)


def full_size(out_dir, t):
    """Reference forward / backward at BASELINE configs 1 and 2, and the reference backward's own run-to-run spread and
    distance from the fp64 oracle (four runs: its fp32 atomics accumulate in an order the hardware picks)."""
    g = {}
    for name, cfg in cases.full_size_configs():
        P, s, sr = cfg["pooled"], cfg["scale"], cfg["sampling_ratio"]
        f, r, dy = cases.full_size_case(cfg)
        out = G.roi_align_forward(t(f), t(r), P, P, s, sr).cpu().numpy()
        dx = G.roi_align_backward(t(dy), t(r), cfg["shape"], P, P, s, sr).cpu().numpy()
        io, idx = _sample(out, 11), _sample(dx, 12, nonzero=True)
        g.update({name + "/out_idx": io, name + "/out": out.reshape(-1)[io], name + "/dx_idx": idx, name + "/dx": dx.reshape(-1)[idx]})
    np.savez_compressed(os.path.join(out_dir, "roi_align_full_size.npz"), **g)
    g = {}
    for name, (shape, s, P, sr, r, seed) in cases.spread_cases().items():
        r = r.astype(np.float32)
        dy = np.random.RandomState(seed).standard_normal((r.shape[0], shape[1], P, P)).astype(np.float32)
        ref64 = O.roi_align_backward(dy, r, shape, P, P, s, sr, acc64=True)
        runs = [G.roi_align_backward(t(dy), t(r), shape, P, P, s, sr).cpu().numpy() for _ in range(4)]
        idx = _sample(runs[0], 13, nonzero=True)
        g.update({name + "/reference_run_to_run_max_abs": np.float64(max(float(np.max(np.abs(x - runs[0]))) for x in runs[1:])),
                  name + "/reference_vs_fp64_max_abs": np.float64(max(float(np.max(np.abs(x - ref64))) for x in runs)),
                  name + "/run0_idx": idx, name + "/run0": runs[0].reshape(-1)[idx]})
    np.savez_compressed(os.path.join(out_dir, "roi_align_bwd_spread.npz"), **g)


def geometry(out_dir, t):
    """The reference kernel's forward and dX on the rectangular-bin cases of tests/geometry_cases.py, from its sm_90a build
    (roi_align_geometry_sm90a.npz): a fixed, seeded sample of output positions and of non-zero dX positions per case."""
    from tests import geometry_cases as GC
    g = {}
    for i, name in enumerate(GC.RECT_CASES):
        c, f, r, dy = GC.geometry_case(name)
        PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
        out = G.roi_align_forward(t(f), t(r), PH, PW, s, sr).cpu().numpy()
        dx = G.roi_align_backward(t(dy), t(r), c["shape"], PH, PW, s, sr).cpu().numpy()
        io, idx = GC.golden_positions(out.size, 100 + i), GC.golden_positions(dx.size, 200 + i, nonzero_of=dx)
        g.update({name + "/out_idx": io, name + "/out": out.reshape(-1)[io], name + "/dx_idx": idx, name + "/dx": dx.reshape(-1)[idx]})
    np.savez_compressed(os.path.join(out_dir, "roi_align_geometry_sm%d%da.npz" % torch.cuda.get_device_capability()), **g)


def main(out_dir, steps=None):
    os.makedirs(out_dir, exist_ok=True)
    assert torch.cuda.is_available() and G.available()
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    if steps == ["geometry"]:
        geometry(out_dir, t)
        print("golden written to", out_dir, sorted(os.listdir(out_dir)))
        return
    xfrom = {}
    for name in sorted(cases.ROI_CASES):
        c, f, r, dy = cases.roi_case(name)
        P, s, sr = c["P"], c["scale"], c["sr"]
        F, Rr, DY = t(f), t(r), t(dy)
        out = G.roi_align_forward(F, Rr, P, P, s, sr)
        dx = G.roi_align_backward(DY, Rr, c["shape"], P, P, s, sr)
        np.savez_compressed(os.path.join(out_dir, "roi_align_xfrom_%s.npz" % name), out=out.cpu().numpy(), dx=dx.cpu().numpy())
        xfrom.update({name + "/out": out.cpu().numpy(), name + "/dx": dx.cpu().numpy()})
        lo = G.roi_align_legacy_forward(F, Rr, P, P, s)
        ldx = G.roi_align_legacy_backward(DY, Rr, c["shape"], P, P, s)
        po, am = G.roi_pool_forward(F, Rr, P, P, s)
        pdx = G.roi_pool_backward(DY, am, Rr, c["shape"], P, P, s)
        np.savez_compressed(os.path.join(out_dir, "legacy_pool_%s.npz" % name), legacy_out=lo.cpu().numpy(),
                            legacy_dx=ldx.cpu().numpy(), pool_out=po.cpu().numpy(), pool_argmax=am.cpu().numpy(),
                            pool_dx=pdx.cpu().numpy())
    img, grid, go = cases.crop_case()
    I, Gd, GO = t(img), t(grid), t(go)
    out = G.roi_crop_forward(I, Gd)
    gi, gg = G.roi_crop_backward(I, Gd, GO)
    np.savez_compressed(os.path.join(out_dir, "roi_crop.npz"), out=out.cpu().numpy(), grad_img=gi.cpu().numpy(),
                        grad_grid=gg.cpu().numpy())
    np.savez_compressed(os.path.join(out_dir, "roi_align_xfrom_sm%d%da.npz" % torch.cuda.get_device_capability(dev)), **xfrom)
    keeps = {}
    for n in cases.NMS_SIZES:
        keeps["keep_%d" % n] = G.nms_gpu(t(cases.nms_case(n)), 0.7).cpu().numpy().reshape(-1).astype(np.int32)
    np.savez_compressed(os.path.join(out_dir, "nms.npz"), **keeps)
    full_size(out_dir, t)
    geometry(out_dir, t)
    torch.cuda.synchronize()
    print("golden written to", out_dir, sorted(os.listdir(out_dir)))


if __name__ == "__main__":
    if len(sys.argv) not in (2, 3) or sys.argv[2:] not in ([], ["geometry"]):
        raise SystemExit("usage: python tests/golden/make_golden.py OUT_DIR [geometry]")
    main(sys.argv[1], sys.argv[2:] or None)
