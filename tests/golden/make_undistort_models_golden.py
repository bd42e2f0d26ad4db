"""Writes golden/opencv_undistort_models.npz: cv2.undistortPoints(pts, K, D, None, K) -- the call Frame::UndistortKeyPoints
and ComputeImageBounds make (reference src/Frame.cc:289-350) -- on every camera model of camera_domain_scenes.py and its
points.  A separate file, so that opencv_undistort.npz stays byte-identical.  Needs python-cv2 (4.x); the tests only read
the vectors.  Run from the repository root: python tests/golden/make_undistort_models_golden.py"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import camera_domain_scenes as S  # noqa: E402


def main():
    out = {"cv2_version": np.array(cv2.__version__)}
    for cam in S.CAMERAS:
        pts = S.points(cam)
        D = cam.dist if not cam.four else cam.dist[:4]
        out["pts/" + cam.name] = pts
        out["out/" + cam.name] = cv2.undistortPoints(pts.reshape(-1, 1, 2), cam.K, D, None, cam.K).reshape(-1, 2)
    path = os.path.join(HERE, "opencv_undistort_models.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "cv2", cv2.__version__)


if __name__ == "__main__":
    main()
