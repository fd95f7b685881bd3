"""Regenerate tests/golden/occupancy_cv2.npz: occupancy grids and what OpenCV's distanceTransform makes of them (in
cells, before the recipe's multiply by the resolution), so that tests/test_occupancy_maps.py checks the transform
against the reference's own recipe without needing cv2.

The recipe is the reference benchmark's (src/test/path_optimizer_benchmark.cpp:28-43):
    cv::distanceTransform(binary, dist, CV_DIST_L2, CV_DIST_MASK_PRECISE); dist *= resolution
with binary = 0 at obstacles.  Grids: seeded random ones of several shapes and densities, a single corner obstacle, a
border, and one grid with no obstacle.  Needs opencv-python (cv2).

    python tests/golden/make_golden_occupancy.py
"""
import os

import cv2
import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "occupancy_cv2.npz")


def grids():
    rng = np.random.default_rng(20261016)
    out = []
    for rows, cols, p in ((37, 53, 0.01), (64, 48, 0.1), (90, 31, 0.3), (17, 120, 0.002), (128, 128, 0.02),
                          (1, 75, 0.05), (60, 1, 0.05), (45, 45, 0.7)):
        occ = (rng.random((rows, cols)) >= p).astype(np.uint8)
        if (occ == 0).sum() == 0:
            occ[rows // 2, cols // 2] = 0
        out.append(occ)
    corner = np.ones((50, 70), np.uint8)
    corner[-1, -1] = 0
    border = np.ones((40, 33), np.uint8)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = 0
    out += [corner, border, np.ones((23, 29), np.uint8)]   # the last one has no obstacle
    return out


def main():
    occs = grids()
    data = {}
    for k, occ in enumerate(occs):
        data[f"occ_{k}"] = occ
        data[f"cv2_{k}"] = cv2.distanceTransform(occ, cv2.DIST_L2, cv2.DIST_MASK_PRECISE)
    data["n"] = np.int32(len(occs))
    data["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **data)
    print(f"wrote {OUT} ({len(occs)} grids, OpenCV {cv2.__version__})")


if __name__ == "__main__":
    main()
