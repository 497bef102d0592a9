"""Write tests/golden/jpeg.npz: for every case of tests/jpeg_cases.py its JPEG bytes, cv2.imdecode's pixels (IMREAD_COLOR) for
cases of at most jpeg_cases.SMALL pixels, else their SHA-256, and the status the device decoder reports.

    python tests/golden/make_golden_jpeg.py

Runs on the CPU with cv2 (the decoder whose pixels the package reproduces) and PIL (the EXIF and progressive writer)."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import jpeg_cases as cases  # noqa: E402


def main():
    import cv2
    out = {}
    for k, name in enumerate(cases.NAMES):
        c = cases.CASES[name]
        data = cases.encode(c, seed=1000 + k)
        im = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        assert im is not None, name
        out[name + "/jpeg"] = np.frombuffer(data, np.uint8)
        out[name + "/shape"] = np.array(im.shape, np.int64)
        if im.shape[0] * im.shape[1] <= cases.SMALL:
            out[name + "/pixels"] = im
        out[name + "/sha256"] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(im).tobytes()).hexdigest().encode(), np.uint8)
        out[name + "/status"] = np.array(c["status"], np.int64)
    path = os.path.join(ROOT, "tests", "golden", "jpeg.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d cases, %d bytes)" % (path, len(cases.NAMES), os.path.getsize(path)))


if __name__ == "__main__":
    main()
