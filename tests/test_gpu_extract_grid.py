"""GPU parity at the bench's batch shape: 64 frames of 1920x1080 in one call, where the FAST kernel runs one CTA per
(tile, frame), 55,296 of them.  Frames spread over the batch equal the CPU oracle, in both batch schedules."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200.synth import shifted_frame, textured_frame

pytestmark = pytest.mark.gpu

W, H, B, NF = 1920, 1080, 64, 2000


def test_1080p_batch_of_64_matches_oracle(gpu_required):
    base = textured_frame(W, H, seed=21)
    frames = np.stack([base] + [shifted_frame(base, 3 * i, 2 * i, seed=100 + i) for i in range(1, B)])
    ex = fe.ORBextractor(NF, 1.2, 8, fe.FAST_SCORE, 20)
    k0, d0, c0 = ex.extract_batch(frames)          # chunked: the upload and the whole chain per quarter of the batch
    ex.set_batch_mode(1)
    k1, d1, c1 = ex.extract_batch(frames)          # phased: one FAST launch over all 64 frames
    ex.close()
    assert np.array_equal(c0, c1) and c0.min() > 0
    for f in range(B):
        assert np.array_equal(k0[f, :c0[f]], k1[f, :c1[f]]) and np.array_equal(d0[f, :c0[f]], d1[f, :c1[f]]), f
    p = O.make_params(NF, 1.2, 8, 1, 20)
    for f in (0, 21, 42, B - 1):
        rc, ok, od, _ = O.extract(p, frames[f])
        assert rc == 0 and c0[f] == len(ok), (f, c0[f], len(ok))
        gk = k0[f, :c0[f]]
        for name in ("x", "y", "size", "response", "octave", "class_id"):
            assert np.array_equal(gk[name], ok[name]), (f, name)
        assert np.max(np.abs(gk["angle"] - ok["angle"]), initial=0.0) <= 1e-4
        assert np.array_equal(d0[f, :c0[f]], od), f
