"""Generate tests/golden/legacy_pool_crop_sm90a.npz from the REFERENCE's own RoIPool, legacy RoIAlign and RoICrop kernels
(oracle/_ref/*.so, built by `make -C oracle ref REFERENCE=<reference checkout>` from its unmodified sources for sm_90a).
Needs an H100:

    python tests/golden/make_golden_legacy_pool_crop.py OUT_DIR      # then copy OUT_DIR/*.npz into tests/golden/

Inputs are the seeded cases of tests/legacy_pool_crop_cases.py whose `golden` flag is set; only the reference OUTPUTS are
stored.  Results the kernels claim bit-exact (legacy RoIAlign forward, RoIPool output / argmax / dX, RoICrop output) are
stored as the sha256 of the complete array (legacy_pool_crop_cases.digest) plus a seeded sample of positions; the image
gradients the reference sums with fp32 atomics as a sample of non-zero positions.  The RoIPool argmax sample is drawn
from the whole array.  Every case has valid batch indices and maps of at least 2 x 2: the reference kernels read and
write outside their tensors otherwise, so the tests pin those cases against the oracle only.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import gpu_ref as G                  # noqa: E402
from tests import legacy_pool_crop_cases as LC   # noqa: E402


def pool_legacy(t, g):
    for i, (name, c) in enumerate(sorted(LC.POOL_LEGACY_CASES.items())):
        if not c["golden"]:
            continue
        N, C, H, W = c["shape"]
        assert H >= 2 and W >= 2
        f, r, dy = LC.roi_case(c)
        assert np.all((r[:, 0] >= 0) & (r[:, 0] < N))
        PH, PW, s = c["PH"], c["PW"], c["scale"]
        F, Rr, DY = t(f), t(r), t(dy)
        lo = G.roi_align_legacy_forward(F, Rr, PH, PW, s).cpu().numpy()
        ldx = G.roi_align_legacy_backward(DY, Rr, c["shape"], PH, PW, s).cpu().numpy()
        po, am = G.roi_pool_forward(F, Rr, PH, PW, s)
        pdx = G.roi_pool_backward(DY, am, Rr, c["shape"], PH, PW, s).cpu().numpy()
        po, am = po.cpu().numpy(), am.cpu().numpy()
        k = "pl/%s/" % name
        li = LC.golden_positions(ldx.size, 300 + i, nonzero_of=ldx)        # NaN counts as non-zero (P - 1 = 0)
        ai = LC.golden_positions(am.size, 400 + i)
        pi = LC.golden_positions(pdx.size, 500 + i, nonzero_of=pdx)
        g.update({k + "legacy_out_sha256": np.array(LC.digest(lo)),
                  k + "legacy_dx_idx": li, k + "legacy_dx": ldx.reshape(-1)[li],
                  k + "pool_out_sha256": np.array(LC.digest(po)),
                  k + "pool_argmax_sha256": np.array(LC.digest(am)),
                  k + "pool_argmax_idx": ai, k + "pool_argmax": am.reshape(-1)[ai],
                  k + "pool_dx_sha256": np.array(LC.digest(pdx)),
                  k + "pool_dx_idx": pi, k + "pool_dx": pdx.reshape(-1)[pi]})
        print(name, "legacy NaN outputs:", int(np.isnan(lo).sum()), "pool argmax -1:", int((am < 0).sum()))


def crop(t, g):
    for i, (name, c) in enumerate(sorted(LC.CROP_CASES.items())):
        if not c["golden"]:
            continue
        N = c["shape"][0]
        assert c["R"] % N == 0
        img, grid, go = LC.crop_case(c)
        I, Gd, GO = t(img), t(grid), t(go)
        out = G.roi_crop_forward(I, Gd).cpu().numpy()
        gi, gg = G.roi_crop_backward(I, Gd, GO)
        gi, gg = gi.cpu().numpy(), gg.cpu().numpy()
        k = "crop/%s/" % name
        oi = LC.golden_positions(out.size, 600 + i)
        gix = LC.golden_positions(gi.size, 700 + i, nonzero_of=gi)
        g.update({k + "out_sha256": np.array(LC.digest(out)), k + "out_idx": oi, k + "out": out.reshape(-1)[oi],
                  k + "grad_img_idx": gix, k + "grad_img": gi.reshape(-1)[gix],
                  k + "grad_grid_nonzero": np.int64(np.count_nonzero(gg))})


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    assert torch.cuda.is_available() and G.available()
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    g = {}
    pool_legacy(t, g)
    crop(t, g)
    torch.cuda.synchronize()
    path = os.path.join(out_dir, "legacy_pool_crop_sm%d%da.npz" % torch.cuda.get_device_capability(dev))
    np.savez_compressed(path, **g)
    print("golden written to", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python tests/golden/make_golden_legacy_pool_crop.py OUT_DIR")
    main(sys.argv[1])
