"""Moment-designed frames for the extractor's orientation and steered BRIEF, and a vectorised restatement of both with the
wrong variants the tests name (numpy and the oracle's primitives only; used by test_oracle_orient_domain.py and
test_gpu_orient_domain.py).

Restatement: IC_Angle's angle from (m01, m10) through cv::fastAtan2 (ORBextractor.cc:150), the angle -> (a, b) map and the 512
rounded (rx, ry) offsets of computeOrbDescriptor (:159-167).  Every binary32 operation is rounded on its own; nothing is
contracted into an FMA; cos / sin are glibc's double functions narrowed to float (the oracle's TRIG_RN).  VARIANTS are the
ways a kernel can get this subtly wrong:

  gt_branch        `ax > ay` for `ax >= ay` in fastAtan2 (|m01| == |m10|, and (0, 0) where eps decides)
  fma_poly         the polynomial contracted into three FMAs
  fma_rot          the rotated coordinate as fmaf(px, b, py * a) and fmaf(px, a, -(py * b))
  half_away        roundf: halves away from zero instead of to even
  floor_half       (int)floorf(v + 0.5f)
  libmf            cosf / sinf (the oracle's TRIG_LIBMF)
  blurred_outside  samples outside the image read the blurred level (reflected) instead of the reflected, unblurred frame

A designed keypoint is an isolated level-0 FAST corner: one pixel `C0_DELTA` off a flat 9x9 square (so its ring and its
neighbours' rings are flat), inside a radius-15 disk whose other pixels are chosen so that IC_Angle's moments hit a target
exactly.  Textured targets use a clipped ramp over small noise, solved by Newton and finished with unit steps on the u = 0
column and the v = 0 row; saturated targets use a 0 / 255 half disk on a 0 background with the corner pixel (255) on the
dark side of the edge, which reaches the bound 255 * 2448 = 624240 exactly on an axis.
"""
import ctypes as C
import ctypes.util
import math
import os

import numpy as np

import oracle as O

F32, F64 = np.float32, np.float64
E = O.EDGE
VARIANTS = ("gt_branch", "fma_poly", "fma_rot", "half_away", "floor_half", "libmf", "blurred_outside")

_INC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "orbfe_brief_pattern.inc")
PATTERN = np.array([int(t) for t in open(_INC).read().split("*/")[1].replace("\n", " ").split(",") if t.strip()],
                   np.int32).reshape(512, 2)          # point 2i, 2i+1 = pair i; (x, y)
PX, PY = PATTERN[:, 0].astype(F32), PATTERN[:, 1].astype(F32)

SCALE = F32(180.0 / math.pi)
P1, P3 = F32(0.9997878412794807) * SCALE, F32(-0.3258083974640975) * SCALE
P5, P7 = F32(0.1555786518463281) * SCALE, F32(-0.04432655554792128) * SCALE
EPS = F32(2.2204460492503131e-16)                      # (float)DBL_EPSILON
FACTOR_PI = F32(math.pi / 180.0)                       # (float)(CV_PI / 180.f)
HALF_DISK_BOUND = 255 * 2448                           # |m| of a saturated half disk


# ---------------------------------------------------------------------------------------------------------------------
# restatement
# ---------------------------------------------------------------------------------------------------------------------
def fma32(x, y, z):
    """fmaf: x * y + z rounded once to binary32 (float32 arrays).  The product is exact in double; the sum is split into
    s + e exactly (TwoSum), and a double s that falls exactly halfway between two floats is resolved by the sign of e."""
    x, y, z = (np.asarray(t, F32) for t in np.broadcast_arrays(x, y, z))
    p, zd = x.astype(F64) * y.astype(F64), z.astype(F64)
    s = p + zd
    bb = s - p
    e = (p - (s - bb)) + (zd - bb)
    r = s.astype(F32)
    rd = r.astype(F64)
    n = np.nextafter(r, np.where(s > rd, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (s != rd) & (2 * s == rd + n.astype(F64))
    return np.where(mid & (e != 0) & ((e > 0) == (s > rd)), n, r)


def fast_atan2(y, x, variant=None):
    """cv::fastAtan2 in degrees on float32 arrays."""
    y, x = np.asarray(y, F32), np.asarray(x, F32)
    ax, ay = np.abs(x), np.abs(y)
    big = (ax > ay) if variant == "gt_branch" else (ax >= ay)
    c = np.where(big, ay, ax) / (np.where(big, ax, ay) + EPS)
    c2 = c * c
    if variant == "fma_poly":
        t = fma32(fma32(fma32(P7, c2, P5), c2, P3), c2, P1) * c
    else:
        t = (((P7 * c2 + P5) * c2 + P3) * c2 + P1) * c
    a = np.where(big, t, F32(90) - t)
    a = np.where(x < 0, F32(180) - a, a)
    return np.where(y < 0, F32(360) - a, a).astype(F32)


def angle_of(m01, m10, variant=None):
    return fast_atan2(np.asarray(m01).astype(F32), np.asarray(m10).astype(F32), variant)


_libm = None


def _cosf_sinf():
    global _libm
    if _libm is None:
        _libm = C.CDLL(ctypes.util.find_library("m"))
        for f in (_libm.cosf, _libm.sinf):
            f.restype, f.argtypes = C.c_float, [C.c_float]
    return _libm.cosf, _libm.sinf


def trig(angle, variant=None):
    """(a, b) = (cos, sin) of angle * factorPI as float32 arrays: (float)cos((double)th), or cosf / sinf for libmf."""
    th = np.asarray(angle, F32).ravel() * FACTOR_PI
    if variant == "libmf":
        cf, sf = _cosf_sinf()
        a = np.array([cf(float(t)) for t in th], F32)
        b = np.array([sf(float(t)) for t in th], F32)
    else:
        a = np.array([math.cos(float(t)) for t in th], F32)
        b = np.array([math.sin(float(t)) for t in th], F32)
    return a, b


def rotated(a, b, variant=None):
    """The unrounded float32 rotated pattern (fx, fy), each [n, 512]."""
    a, b = np.asarray(a, F32)[:, None], np.asarray(b, F32)[:, None]
    if variant == "fma_rot":
        return fma32(PX, a, -(PY * b)), fma32(PX, b, PY * a)
    return PX * a - PY * b, PX * b + PY * a


def cv_round(v, variant=None):
    if variant == "half_away":
        return (np.sign(v) * np.floor(np.abs(v).astype(F64) + 0.5)).astype(np.int64)
    if variant == "floor_half":
        return np.floor(v + F32(0.5)).astype(np.int64)
    return np.rint(v).astype(np.int64)


def offsets(a, b, variant=None):
    """The 512 rounded sample offsets (rx, ry), each [n, 512] int."""
    fx, fy = rotated(a, b, variant)
    return cv_round(fx, variant), cv_round(fy, variant)


def ties(a, b):
    """Per keypoint, the number of rotated coordinates (of 1024) that are exact halves, split into classes
    {(sign, parity of the integer part): count}."""
    fx, fy = rotated(a, b)
    v = np.concatenate([fx, fy], axis=1).astype(F64)
    tie = (v - np.floor(v)) == 0.5
    ip = np.trunc(v).astype(np.int64)
    out = []
    for k in range(len(v)):
        cls = {}
        for s, par in zip(np.where(v[k][tie[k]] > 0, "+", "-"), np.abs(ip[k][tie[k]]) % 2):
            key = s + ("odd" if par else "even")
            cls[key] = cls.get(key, 0) + 1
        out.append(cls)
    return out


DISK = np.array([(u, v) for v in range(-15, 16) for u in range(-15, 16) if abs(u) <= O.UMAX[abs(v)]], np.int64)
DU, DV = DISK[:, 0], DISK[:, 1]
assert int(DV[DV > 0].sum()) * 255 == HALF_DISK_BOUND and int(DU[DU > 0].sum()) * 255 == HALF_DISK_BOUND


def moments(padded, xs, ys, pad=E):
    """IC_Angle's (m01, m10) of keypoints (xs, ys) of a padded level image (int arrays)."""
    xs, ys = np.asarray(xs, np.int64), np.asarray(ys, np.int64)
    vals = padded[ys[:, None] + pad + DV[None, :], xs[:, None] + pad + DU[None, :]].astype(np.int64)
    return (vals * DV).sum(axis=1), (vals * DU).sum(axis=1)


def describe(buf, xs, ys, rx, ry, pad=E):
    """Steered BRIEF bytes [n, 32] from a padded buffer (interior blurred)."""
    xs, ys = np.asarray(xs, np.int64)[:, None], np.asarray(ys, np.int64)[:, None]
    t = buf[ys + pad + ry, xs + pad + rx]
    bits = (t[:, 0::2] < t[:, 1::2]).astype(np.uint8).reshape(-1, 32, 8)[:, :, ::-1]
    return np.packbits(bits, axis=2).reshape(-1, 32)


def level_coords(p, kps):
    """Level coordinates (ints) of reported keypoints: level 0 as is, else x = rint(kx / scale) with f32(x * scale) == kx."""
    oc = kps["octave"]
    s = np.array([p.scale[int(l)] for l in oc], F32)
    x = np.where(oc == 0, kps["x"], np.rint(kps["x"] / s)).astype(np.int64)
    y = np.where(oc == 0, kps["y"], np.rint(kps["y"] / s)).astype(np.int64)
    assert np.array_equal(np.where(oc == 0, x.astype(F32), x.astype(F32) * s), kps["x"])
    assert np.array_equal(np.where(oc == 0, y.astype(F32), y.astype(F32) * s), kps["y"])
    return x, y


def restate(p, dump, kps, variant=None):
    """Angles and descriptors of the oracle's keypoints `kps` from its dump (level images, blurred levels), under a variant
    (None: the rule).  Returns (angles float32 [n], descriptors uint8 [n, 32])."""
    xs, ys = level_coords(p, kps)
    ang = np.zeros(len(kps), F32)
    desc = np.zeros((len(kps), 32), np.uint8)
    for l in np.unique(kps["octave"]):
        k = np.flatnonzero(kps["octave"] == l)
        m01, m10 = moments(dump["levels"][l].astype(np.int64), xs[k], ys[k])
        ang[k] = angle_of(m01, m10, variant)
        a, b = trig(ang[k], variant)
        rx, ry = offsets(a, b, variant)
        buf = dump["blurred"][l]
        if variant == "blurred_outside":
            buf = O.reflect101_pad(buf[E:-E, E:-E], E)
        desc[k] = describe(buf, xs[k], ys[k], rx, ry)
    return ang, desc


def outside_samples(xs, ys, w, h, angles):
    """Per keypoint, how many of its 512 samples fall outside the w x h level."""
    a, b = trig(angles)
    rx, ry = offsets(a, b)
    sx, sy = np.asarray(xs)[:, None] + rx, np.asarray(ys)[:, None] + ry
    return ((sx < 0) | (sx >= w) | (sy < 0) | (sy >= h)).sum(axis=1)


# ---------------------------------------------------------------------------------------------------------------------
# bounded search for tie pairs and trig-split pairs (how the constants below were found)
# ---------------------------------------------------------------------------------------------------------------------
def search(n=100000, bound=200000, seed=7, chunk=10000):
    """Random (m01, m10) in [-bound, bound]^2.  Returns {"ties": {class: [(m01, m10)]}, "trig": [(m01, m10)],
    "fma_rot": [...]}: pairs whose rotated pattern has an exact half of that class, pairs whose rounded offsets change
    under cosf / sinf, and pairs whose rounded offsets change under the contracted rotation."""
    rng = np.random.default_rng(seed)
    m = rng.integers(-bound, bound + 1, (n, 2))
    out = {"ties": {}, "trig": [], "fma_rot": []}
    for c0 in range(0, n, chunk):
        mm = m[c0:c0 + chunk]
        ang = angle_of(mm[:, 0], mm[:, 1])
        a, b = trig(ang)
        rx, ry = offsets(a, b)
        al, bl = trig(ang, "libmf")
        split = np.flatnonzero((al != a) | (bl != b))
        if len(split):
            lx, ly = offsets(al[split], bl[split])
            hit = ((lx != rx[split]) | (ly != ry[split])).any(axis=1)
            out["trig"] += [tuple(int(t) for t in mm[i]) for i in split[hit]]
        fx, fy = offsets(a, b, "fma_rot")
        for i in np.flatnonzero(((fx != rx) | (fy != ry)).any(axis=1)):
            out["fma_rot"].append(tuple(int(t) for t in mm[i]))
        fxr, fyr = rotated(a, b)
        v = np.concatenate([fxr, fyr], axis=1)
        for i in np.flatnonzero(((v.astype(F64) - np.floor(v)) == 0.5).any(axis=1)):
            for cls in ties(a[i:i + 1], b[i:i + 1])[0]:
                out["ties"].setdefault(cls, []).append(tuple(int(t) for t in mm[i]))
    return out


# TIE_PAIRS: search() (10^5 pairs), the first two pairs of each class not already taken.  TRIG_PAIRS: search(n=2 * 10**6) and
# search(n=4 * 10**5, seed=11) -- cosf / sinf differ from the correctly rounded values on ~1.3% of angles, but move a
# rounded offset for only about one pair in 10^5.  test_oracle_orient_domain.py re-derives what each pair does.
TIE_PAIRS = {"+even": [(-154278, 191105), (74807, -181598)], "+odd": [(12775, 1406), (16527, 35853)],
             "-even": [(99477, -19397), (-160554, 125390)], "-odd": [(11397, 34409), (-26329, -192080)]}
# Pairs whose angle changes when the polynomial is contracted (1.75% of random pairs do).
FMA_POLY_PAIRS = [(119076, 137693), (104825, -121936), (179887, -147742), (-190792, -138406)]
TRIG_PAIRS = [(-66416, 101771), (90708, 59751), (3269, 1244), (-149793, -106820), (-118129, 140187), (36726, 137711),
              (-128318, 196625)]


# ---------------------------------------------------------------------------------------------------------------------
# disk designs
# ---------------------------------------------------------------------------------------------------------------------
BG = 128
C0_DELTA = 60             # the corner pixel's contrast (FAST score 59 at the default threshold 20)
ZONE = 4                  # flat square |u|, |v| <= 4 around the corner


def _fix(vals, r, coord, other, lo=0, hi=255):
    """Bring residual r of sum(coord * vals) to zero with unit steps on pixels where `other` == 0 and |coord| >= 5."""
    idx = np.flatnonzero((other == 0) & (np.abs(coord) >= 5))
    idx = idx[np.argsort(-np.abs(coord[idx]))]
    while r:
        done = False
        for i in idx:
            for st in (1, -1):
                d = coord[i] * st
                if abs(r - d) < abs(r) and lo <= vals[i] + st <= hi:
                    vals[i] += st
                    r -= d
                    done = True
                    break
            if done:
                break
        if done:
            continue
        # |r| < 5: +1 at |coord| = 5 + |r| and -1 at |coord| = 5 on one side
        for sgn in (1, -1):
            i1 = np.flatnonzero((other == 0) & (coord == sgn * (5 + abs(r))))[0]
            i0 = np.flatnonzero((other == 0) & (coord == sgn * 5))[0]
            st = 1 if r * sgn > 0 else -1
            if lo <= vals[i1] + st <= hi and lo <= vals[i0] - st <= hi:
                vals[i1] += st
                vals[i0] -= st
                r = 0
                break
        else:
            raise ValueError("no headroom for the residual")
    return vals


def flip_stamp(m01, m10, variant):
    """{(u, v): value} that makes the variant flip a descriptor bit of a keypoint with moments (m01, m10): around the first
    sample the variant moves (RN offset r, the variant's r'), a 0 / 255 step edge between r and r' (blurred about 100 at r
    and 155 at r'), and 128 around its pair partner where that does not overlap the edge.  Every stamped pixel is within
    3 px of a sample and outside the flat square; None when no moved sample allows that."""
    ang = angle_of([m01], [m10])
    a, b = trig(ang)
    rx, ry = offsets(a, b)
    av, bv = trig(angle_of([m01], [m10], variant), variant)
    vx, vy = offsets(av, bv, variant)
    for j in np.flatnonzero((rx[0] != vx[0]) | (ry[0] != vy[0])):
        p, q, k = (int(rx[0, j]), int(ry[0, j])), (int(vx[0, j]), int(vy[0, j])), j ^ 1
        part = (int(rx[0, k]), int(ry[0, k]))
        box = [(u, v) for u in range(min(p[0], q[0]) - 3, max(p[0], q[0]) + 4)
               for v in range(min(p[1], q[1]) - 3, max(p[1], q[1]) + 4)]
        pbox = [(u, v) for u in range(part[0] - 3, part[0] + 4) for v in range(part[1] - 3, part[1] + 4)]
        pbox = [uv for uv in pbox if uv not in set(box)]
        if any(max(abs(u), abs(v)) <= ZONE for u, v in box + pbox):
            continue
        d = (q[0] - p[0], q[1] - p[1])
        st = {(u, v): (255 if (u - p[0]) * d[0] + (v - p[1]) * d[1] > 0 else 0) for u, v in box}
        st.update({uv: 128 for uv in pbox})
        return st
    return None


def ramp_disk(m01, m10, rng, c0=BG + C0_DELTA, fixed=None):
    """Disk values (aligned with DISK) on a BG background whose moments are exactly (m01, m10); `fixed` {(u, v): value}
    pins disk pixels (those outside the disk are the caller's to write)."""
    zone = (np.abs(DU) <= ZONE) & (np.abs(DV) <= ZONE)
    pin = np.zeros(len(DISK), bool)
    pinned = np.zeros(len(DISK), np.int64)
    for i, (u, v) in enumerate(DISK):
        if fixed and (int(u), int(v)) in fixed:
            pin[i], pinned[i] = True, fixed[(int(u), int(v))]
    free = ~zone & ~pin
    t01, t10 = m01 - int((pinned * DV).sum()), m10 - int((pinned * DU).sum())
    base = BG + rng.integers(-6, 7, len(DISK)).astype(F64)
    u, v = DU[free].astype(F64), DV[free].astype(F64)
    A = B = 0.0
    for _ in range(60):
        raw = base[free] + A * v + B * u
        val = np.clip(raw, 0, 255)
        inr = ((raw > 0) & (raw < 255)).astype(F64)
        r = np.array([t01 - (v * val).sum(), t10 - (u * val).sum()])
        if np.abs(r).max() < 0.5:
            break
        J = np.array([[(v * v * inr).sum(), (u * v * inr).sum()], [(u * v * inr).sum(), (u * u * inr).sum()]])
        dA, dB = np.linalg.solve(J, r)
        A, B = A + dA, B + dB
    vals = np.full(len(DISK), BG, np.int64)
    vals[free] = np.clip(np.rint(base[free] + A * v + B * u), 0, 255).astype(np.int64)
    vals[(DU == 0) & (DV == 0)] = c0
    vals[pin] = pinned[pin]
    vals = _fix(vals, m01 - int((vals * DV).sum()), DV, np.where(pin, 1, DU))
    vals = _fix(vals, m10 - int((vals * DU).sum()), DU, np.where(pin, 1, DV))
    assert (int((vals * DV).sum()), int((vals * DU).sum())) == (m01, m10)
    return vals


def half_disk(nu, nv, tweaks=()):
    """Disk values on a 0 background: 255 where nu*u + nv*v > 0, the corner pixel 255, then (u, v, value) tweaks."""
    vals = np.where(nu * DU + nv * DV > 0, 255, 0).astype(np.int64)
    vals[(DU == 0) & (DV == 0)] = 255
    for u, v, val in tweaks:
        vals[(DU == u) & (DV == v)] = val
    return vals


def disk_moments(vals):
    return int((vals * DV).sum()), int((vals * DU).sum())


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
NF, FAST_TH = 2000, 20


def nfeatures(nlevels):
    """2000 over 8 levels, 1500 on one: both keep every designed keypoint, and both give cells the library accepts (more
    features give smaller cells, which it refuses on these small frames)."""
    return NF if nlevels > 1 else 1500


IW, IH = 352, 272                                     # interior frames: 8 x 6 keypoints 40 px apart
SLOTS = [(36 + 40 * i, 36 + 40 * j) for j in range(6) for i in range(8)]
BORDER_WIDTHS = (384, 385, 386, 387)                  # W mod 4 = 0..3; 384 = 3 * 128: the plan's pitch equals W
BORDER_H = 360
BORDER_D = (16, 17, 18, 19, 20, 21, 22)               # distance of a keypoint from the near edge, or W - 1 - x from the far


def _frame(W, H, bg, designs):
    """designs: [(x, y, vals)] or [(x, y, vals, {(u, v): value} outside the disk)].  Returns (image, [(x, y, m01, m10)])."""
    img = np.full((H, W), bg, np.uint8)
    kps = []
    for d in designs:
        x, y, vals = d[:3]
        img[y + DV, x + DU] = vals
        for (u, v), val in (d[3] if len(d) > 3 else {}).items():
            if abs(u) > O.UMAX[min(abs(v), 15)] or abs(v) > 15:
                img[y + v, x + u] = val
        kps.append((x, y) + disk_moments(vals))
    return img, kps


def _ramp_frame(name, targets, seed, W=IW, H=IH, slots=None, flip=None):
    """Textured designs of `targets` at `slots`; with flip = a variant, each keypoint also carries flip_stamp's edge."""
    rng = np.random.default_rng(seed)
    slots = slots or SLOTS
    designs = []
    for k, ((x, y), (m01, m10)) in enumerate(zip(slots, targets)):
        st = flip_stamp(m01, m10, flip) if flip else None
        designs.append((x, y, ramp_disk(m01, m10, rng, BG + (C0_DELTA if k % 2 == 0 else -C0_DELTA), st), st or {}))
    img, kps = _frame(W, H, BG, designs)
    return dict(name=name, img=img, kps=kps)


def _border_designs(W, H):
    """Keypoints BORDER_D px from each edge (left / right columns, top / bottom rows), each with the target among 72
    directions of magnitude 100000 that puts the most samples outside the image."""
    pos = []
    for k, d in enumerate(BORDER_D):
        c = 60 + 40 * k
        pos += [(d, c), (W - 1 - d, c), (c, d), (c, H - 1 - d)]
    dirs = [(int(round(100000 * math.sin(math.radians(t)))), int(round(100000 * math.cos(math.radians(t)))))
            for t in range(0, 360, 5)]
    dang = angle_of([d[0] for d in dirs], [d[1] for d in dirs])
    targets = []
    for x, y in pos:
        n_out = outside_samples(np.full(len(dirs), x), np.full(len(dirs), y), W, H, dang)
        targets.append(dirs[int(np.argmax(n_out))])
    return pos, targets


def scenes():
    """[{name, img, kps: [(x, y, m01, m10)], bg}] -- every designed keypoint of every frame (cached)."""
    global _SCENES
    if _SCENES is not None:
        return _SCENES
    out = []
    K = 150000
    out.append(_ramp_frame("zero_axes_diagonals", [(0, 0)] * 4 + [
        (0, 1), (0, -1), (1, 0), (-1, 0), (0, 777), (0, -777), (777, 0), (-777, 0), (0, K), (0, -K), (K, 0), (-K, 0),
        (1, 1), (1, -1), (-1, 1), (-1, -1), (5000, 5000), (5000, -5000), (-5000, 5000), (-5000, -5000),
        (K, K), (K, -K), (-K, K), (-K, -K), (K + 1, K), (K, K + 1), (-K - 1, K), (K, -K - 1),
        (-1, 300000), (-1, 2), (-2, 1)] + FMA_POLY_PAIRS, seed=1))
    # saturated half disks on a 0 background
    M = HALF_DISK_BOUND
    sat = [half_disk(1, 0), half_disk(0, 1), half_disk(-1, 0), half_disk(0, -1),          # (0, M) (M, 0) (0, -M) (-M, 0)
           half_disk(1, 0, [(0, -1, 1)]),                                                # (-1, M): just below 360
           half_disk(1, 0, [(0, 1, 1)]), half_disk(0, 1, [(-1, 0, 1)]),                  # (1, M), (M, -1)
           half_disk(1, 1), half_disk(-1, 1), half_disk(-1, -1), half_disk(1, -1),       # |m01| == |m10|, four quadrants
           half_disk(1, 1, [(0, -1, 1)]), half_disk(1, 1, [(1, 0, 254)]),                # |m01| = |m10| -+ 1
           half_disk(-1, -1, [(0, 1, 1)]), half_disk(-1, -1, [(-1, 0, 254)])]
    flat = np.zeros(len(DISK), np.int64)
    flat[(DU == 0) & (DV == 0)] = 255
    img, kps = _frame(IW, IH, 0, [(x, y, v) for (x, y), v in zip(SLOTS, sat + [flat])])
    assert kps[0][2:] == (0, M) and kps[4][2:] == (-1, M)
    out.append(dict(name="saturated", img=img, kps=kps))
    out.append(_ramp_frame("ties", [pr for cls in sorted(TIE_PAIRS) for pr in TIE_PAIRS[cls]], seed=2))
    out.append(_ramp_frame("trig_split", TRIG_PAIRS, seed=3, flip="libmf"))
    for W in BORDER_WIDTHS:
        pos, targets = _border_designs(W, BORDER_H)
        out.append(_ramp_frame("border_%d" % W, targets, seed=W, W=W, H=BORDER_H, slots=pos))
    for s in out:
        s["W"], s["H"] = s["img"].shape[1], s["img"].shape[0]
        s["variants"] = SCENE_VARIANTS.get(s["name"], ())
    _SCENES = out
    return out


_SCENES = None
# The variants that change the angle or descriptor of at least one designed keypoint of each scene
# (test_oracle_orient_domain.py derives them again).
SCENE_VARIANTS = {"zero_axes_diagonals": ("gt_branch", "fma_poly"), "saturated": ("gt_branch",),
                  "ties": ("fma_rot", "half_away", "floor_half"), "trig_split": ("half_away", "libmf"),
                  "border_384": ("blurred_outside",), "border_385": ("blurred_outside",),
                  "border_386": ("blurred_outside",), "border_387": ("blurred_outside",)}
