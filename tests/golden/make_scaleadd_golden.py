"""Generates tests/golden/opencv_scaleadd.npz: inputs and python-cv2 outputs of cv2.scaleAdd(src1, alpha, src2) on 3x1
float32 columns, the operation OpenCV evaluates `normal + normali/cv::norm(normali)` with (MapPoint.cc:295; MatOp_AddEx ->
scaleAdd(normali, 1/norm, normal)).  Every case is chosen so that at least one component differs between the product
rounded and then added (src1*alpha rounded to float, + src2 rounded) and the fused result (one rounding).  alpha is a
float value, as scaleAdd casts it to float before use.  Run here (python-cv2 is in the image):
python tests/golden/make_scaleadd_golden.py"""
import os

import cv2
import numpy as np

rng = np.random.default_rng(20261017)
src1, src2, alpha, out = [], [], [], []
while len(src1) < 500:
    a = (rng.standard_normal(3) * rng.choice([1e-3, 1.0, 30.0])).astype(np.float32)
    b = (rng.standard_normal(3) * rng.choice([1e-3, 1.0, 30.0])).astype(np.float32)
    al = np.float32(1.0 / np.sqrt(np.float64(rng.uniform(1e-4, 1e4))))   # (float)(1.0 / cv::norm(d)) magnitudes
    sep = (a * al).astype(np.float32) + b
    fused = (a.astype(np.float64) * np.float64(al) + b.astype(np.float64)).astype(np.float32)
    if np.array_equal(sep, fused):
        continue
    src1.append(a)
    src2.append(b)
    alpha.append(al)
    out.append(cv2.scaleAdd(a.reshape(3, 1), float(al), b.reshape(3, 1)).reshape(3))
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "opencv_scaleadd.npz"), src1=np.array(src1),
                    src2=np.array(src2), alpha=np.array(alpha, np.float32), out=np.array(out, np.float32),
                    cv2_version=np.array(cv2.__version__))
print("wrote opencv_scaleadd.npz with", len(src1), "cases, cv2", cv2.__version__)
