"""Scenes and an independent candidate-set composition for the extractor's domain tests.

Shared by test_oracle_fast_domain.py (CPU: the composition against oracle.extract) and test_gpu_extract_domain.py (the
CUDA extractor against both).  numpy and the oracle's primitives only.

The composition restates ComputeKeyPoints (ORBextractor.cc:549-614) from parts the oracle exports one by one: the oracle's
level images (its dump), its cell grid (O.cell_grid), the reference's window margins (-3 / +6 px around each cell, the last
row and column running to the 16-px border + 3) and cv::FAST with non-maximum suppression on each window (O.fast_detect),
re-run at threshold 7 when it finds <= 3 corners.  When every cell keeps every candidate, the level's keypoints ARE this set.
"""
import numpy as np

import oracle as O
from orb_slam_b200.synth import textured_frame

E = O.EDGE
FT_W, FT_H = 120, 62       # FAST tile of the CUDA kernel (ORBFE_FT_W x ORBFE_FT_H), tiles start at the 16-px border
FALLBACK_TH = 7            # ORBextractor.cc:609-614


# ---------------------------------------------------------------------------------------------------------------------
# composition
# ---------------------------------------------------------------------------------------------------------------------
def cell_windows(p, level, W0, H0, w, h):
    """[(i, j, y0, x0, hh, ww)] of the level's cell windows in interior coordinates (ORBextractor.cc:555-604)."""
    rc, g = O.cell_grid(p, level, W0, H0, w, h)
    assert rc == 0
    out = []
    maxBX, maxBY = w - E, h - E
    for i in range(g.rows):
        iniY = E + i * g.cell_h - 3
        hY = g.cell_h + 6 if i < g.rows - 1 else maxBY + 3 - iniY
        if hY <= 0:
            continue
        for j in range(g.cols):
            iniX = E + j * g.cell_w - 3
            hX = g.cell_w + 6 if j < g.cols - 1 else maxBX + 3 - iniX
            if hX <= 0:
                continue
            out.append((i, j, iniY, iniX, hY, hX))
    return g, out


def level_candidates(p, dump, W0, H0, level):
    """The level's FAST+NMS candidates per the reference's per-cell detection, with the <= 3 -> threshold-7 fallback.

    Returns (xyr, counts): xyr an int array [n, 3] of (x, y, score) in level interior coordinates, cell row-major and
    raster order inside a cell; counts a dict {(i, j): number of candidates at fastTh} (before the fallback)."""
    lev = dump["levels"][level][E:-E, E:-E]
    h, w = lev.shape
    _, wins = cell_windows(p, level, W0, H0, w, h)
    rows, counts = [], {}
    for i, j, y0, x0, hh, ww in wins:
        win = lev[y0:y0 + hh, x0:x0 + ww]
        xs, ys, sc = O.fast_detect(win, p.fast_th)
        counts[(i, j)] = len(xs)
        if len(xs) <= 3:
            xs, ys, sc = O.fast_detect(win, FALLBACK_TH)
        rows.append(np.stack([xs + x0, ys + y0, sc], axis=1))
    xyr = np.concatenate(rows).astype(np.int64) if rows else np.zeros((0, 3), np.int64)
    return xyr, counts


def to_output(p, level, xyr):
    """Level-coordinate candidates as the keypoint fields the extractor reports: (x, y) scaled to level 0 in float32
    (ORBextractor.cc:768-775), response = the FAST score.  Returns a sorted structured array of (x, y, response)."""
    s = np.float32(p.scale[level])
    x = xyr[:, 0].astype(np.float32)
    y = xyr[:, 1].astype(np.float32)
    if level:
        x, y = x * s, y * s
    return triples(x, y, xyr[:, 2].astype(np.float32))


def triples(x, y, r):
    t = np.zeros(len(x), [("x", "<f4"), ("y", "<f4"), ("response", "<f4")])
    t["x"], t["y"], t["response"] = x, y, r
    return np.sort(t, order=("y", "x", "response"))


def octave_triples(kps, level):
    k = kps[kps["octave"] == level]
    return triples(k["x"], k["y"], k["response"])


# ---------------------------------------------------------------------------------------------------------------------
# threshold scenes
# ---------------------------------------------------------------------------------------------------------------------
RING = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
        (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3)]   # (dx, dy) of cv::FAST's 16-ring


def ring_arcs(th, W=320, H=240, seed=0):
    """7x7 patches tiling the frame.  Each has a centre value c and its 16-ring filled from {c-th-1, c-th, c, c+th, c+th+1}
    (clipped to 0..255), with a contiguous arc of 8, 9 or 10 ring pixels drawn only from the two values at th and th+1
    of one polarity: every ring difference sits exactly on, or one past, the FAST threshold."""
    rng = np.random.default_rng(seed * 1000 + th)
    img = np.zeros((H, W), np.uint8)
    for cy in range(3, H - 3, 7):
        for cx in range(3, W - 3, 7):
            bright = bool(rng.integers(0, 2))
            c = int(rng.integers(0, 255 - th)) if bright else int(rng.integers(th + 1, 256))
            img[cy - 3:cy + 4, cx - 3:cx + 4] = c
            vals = np.clip(np.array([c - th - 1, c - th, c, c + th, c + th + 1]), 0, 255)
            arc = (vals[3:] if bright else vals[:2])
            n_arc, start = int(rng.choice([8, 9, 10])), int(rng.integers(0, 16))
            for k, (dx, dy) in enumerate(RING):
                on_arc = (k - start) % 16 < n_arc
                img[cy + dy, cx + dx] = rng.choice(arc) if on_arc else rng.choice(vals)
    return img


def two_tone(th, contrast, W=320, H=240):
    """Single pixels every 13 px on a flat background, two values `contrast` apart: each pixel is a FAST corner of score
    contrast - 1 when contrast > threshold, and nothing else is.  (Shapes of two values give runs of equal scores along
    their edges, which strict NMS removes whole.)"""
    lo = 0 if th >= 127 else 100
    img = np.full((H, W), lo, np.uint8)
    img[5:H - 5:13, 7:W - 5:13] = lo + contrast
    return img


def binary_noise(W=320, H=240, seed=0):
    return (np.random.default_rng(seed).integers(0, 2, (H, W)) * 255).astype(np.uint8)


COUNT_NF, COUNT_NL = 500, 1
COUNT_CELL_A, COUNT_CELL_B = (2, 2), (4, 5)   # cells with exactly 3 and exactly 4 candidates at fastTh


def count_scene(th, W=320, H=240):
    """Isolated single-pixel corners on a flat frame (a single pixel of contrast d is a FAST corner of score d - 1 with no
    corner neighbour).  Cell A holds 3 of contrast th + 1 and cell B 4: exactly 3 and exactly 4 candidates at fastTh, so A
    falls back to threshold 7 and B does not.  For th >= 8 both also hold 2 of contrast exactly th, which only the
    threshold-7 pass sees: A keeps 5 and B keeps 4.  For th <= 6 the threshold-7 pass finds nothing in A: A keeps 0.
    Every other cell is empty (and falls back).  At th = 0 the corners have contrast 2: one of contrast 1 has score 0, and
    cv::FAST's strict non-maximum suppression never keeps a score of 0.  Returns (image, {cell: expected kept})."""
    p = O.make_params(COUNT_NF, 1.2, COUNT_NL, 1, th)
    g = O.cell_grid(p, 0, W, H, W, H)[1]
    bg = 0 if th >= 127 else 128
    img = np.full((H, W), bg, np.uint8)
    offs = [(-6, -5), (0, -5), (6, -5), (-6, 4), (0, 4), (6, 4)]
    expect = {}
    for cell, n_strong in ((COUNT_CELL_A, 3), (COUNT_CELL_B, 4)):
        i, j = cell
        cx, cy = E + j * g.cell_w + g.cell_w // 2, E + i * g.cell_h + g.cell_h // 2
        contrasts = [max(th + 1, 2)] * n_strong + ([th] * 2 if th >= 8 else [])
        for k, d in enumerate(contrasts):
            dx, dy = offs[k]
            sign = 1 if (bg == 0 or k % 2 == 0) else -1
            img[cy + dy, cx + dx] = bg + sign * d
        if n_strong > 3:
            expect[cell] = n_strong
        else:
            expect[cell] = len(contrasts) if th >= 7 else 0
    return img, expect


def threshold_scenes(th):
    """{name: image} for one FAST threshold (320x240 frames)."""
    return {"arcs": ring_arcs(th), "two_tone_th": two_tone(th, th), "two_tone_th1": two_tone(th, th + 1),
            "binary": binary_noise(seed=th), "textured": textured_frame(320, 240, seed=th + 5),
            "count": count_scene(th)[0]}


# ---------------------------------------------------------------------------------------------------------------------
# seam scenes: isolated single-pixel corners in adjacent pairs across every seam of level 0
# ---------------------------------------------------------------------------------------------------------------------
# (W, H, nlevels): detect area Wd = W - 32 with Wd mod 120 in {0, 1, 2, 118, 119}, Hd = H - 32 with Hd mod 62 in {0, 1, 61}
SEAM_GEOMETRIES = [(512, 466, 1), (513, 467, 2), (514, 465, 3), (510, 466, 2), (511, 465, 1)]
SEAM_NF, SEAM_TH, SEAM_BG = 1500, 20, 128


class _Stamps:
    def __init__(self, img):
        self.img = img
        self.pts = []       # (x, y)
        self.pairs = []     # ((x1, y1, d1), (x2, y2, d2)); d signed contrast

    def free(self, x, y, r=4):
        H, W = self.img.shape
        if not (0 <= x < W and 0 <= y < H):
            return False
        return all(max(abs(x - a), abs(y - b)) > r for a, b in self.pts)

    def pair(self, x1, y1, x2, y2, d1, d2):
        if not (self.free(x1, y1) and self.free(x2, y2)):
            return False
        for x, y, d in ((x1, y1, d1), (x2, y2, d2)):
            self.img[y, x] = SEAM_BG + d
            self.pts.append((x, y))
        self.pairs.append(((x1, y1, d1), (x2, y2, d2)))
        return True


def seam_scene(W, H, nl, seed=0):
    """A flat frame with single-pixel corners in adjacent pairs straddling every interior cell seam of level 0 (both
    orientations, unequal and equal contrast), every FAST-tile seam, the 16-px detect border on all four sides, plus pairs
    inside cells.  Returns (image, pairs)."""
    rng = np.random.default_rng(seed + W * 7 + H)
    img = np.full((H, W), SEAM_BG, np.uint8)
    S = _Stamps(img)
    p = O.make_params(SEAM_NF, 1.2, nl, 1, SEAM_TH)
    g = O.cell_grid(p, 0, W, H, W, H)[1]
    cw, ch, rows, cols = g.cell_w, g.cell_h, g.rows, g.cols
    xmax, ymax = W - E, H - E   # detect area is [16, xmax) x [16, ymax)

    def contrasts(equal):
        a = int(rng.integers(25, 90)) * int(rng.choice([-1, 1]))
        if equal:
            return a, a * int(rng.choice([-1, 1]))          # same |contrast|, either polarity: the same FAST score
        b = int(rng.integers(25, 90))
        while b == abs(a):
            b = int(rng.integers(25, 90))
        return a, b * int(rng.choice([-1, 1]))

    def along(lo, hi, step):
        return list(range(lo, hi, step))

    def vpair(x, ys, equal):        # (x-1, y) | (x, y)
        for y in ys:
            if S.pair(x - 1, y, x, y, *contrasts(equal)):
                return

    def hpair(y, xs, equal):        # (x, y-1) / (x, y)
        for x in xs:
            if S.pair(x, y - 1, x, y, *contrasts(equal)):
                return

    # interior cell seams: x = 16 + j*cw, y = 16 + i*ch; the pair sits mid-cell along the seam, one per cell row / column
    for j in range(1, cols):
        x = E + j * cw
        for i in range(rows):
            mid = E + i * ch + ch // 2
            vpair(x, [mid, mid - 3, mid + 3], equal=bool((i + j) % 2))
    for i in range(1, rows):
        y = E + i * ch
        for j in range(cols):
            mid = E + j * cw + cw // 2
            hpair(y, [mid, mid - 3, mid + 3], equal=bool((i + j) % 2))
    # FAST-tile seams (x = 16 + 120k, y = 16 + 62k): several positions each, unequal and equal
    for x in range(E + FT_W, xmax, FT_W):
        for k, y in enumerate(along(E + 9, ymax - 2, 37)):
            vpair(x, [y, y + 5, y + 10], equal=bool(k % 2))
    for y in range(E + FT_H, ymax, FT_H):
        for k, x in enumerate(along(E + 11, xmax - 2, 41)):
            hpair(y, [x, x + 5, x + 10], equal=bool(k % 2))
    # the detect border: the outer pixel (outside the detect area) is the stronger one
    for y in along(E + 20, ymax - 20, 53):
        S.pair(E - 1, y, E, y, 90, 40)
        S.pair(xmax - 1, y + 7, xmax, y + 7, -40, -90)
    for x in along(E + 25, xmax - 25, 59):
        S.pair(x, E - 1, x, E, -90, 40)
        S.pair(x + 7, ymax - 1, x + 7, ymax, 40, 90)
    # pairs inside cells, horizontal, vertical and diagonal neighbours
    for _ in range(6 * cols):
        x, y = int(rng.integers(E + 4, xmax - 4)), int(rng.integers(E + 4, ymax - 4))
        dx, dy = [(1, 0), (0, 1), (1, 1), (1, -1)][int(rng.integers(0, 4))]
        S.pair(x, y, x + dx, y + dy, *contrasts(bool(rng.integers(0, 2))))
    return img, S.pairs


def seam_expected(W, H, nl, pairs):
    """Level-0 keypoints (x, y) the seam scene must give: a pair inside one cell resolves by strict 3x3 NMS (the stronger
    pixel; neither when the contrasts are equal); a pair whose pixels lie in different cells keeps both; a pixel outside
    the detect area is never a keypoint and suppresses nothing.  FAST-tile seams play no part."""
    p = O.make_params(SEAM_NF, 1.2, nl, 1, SEAM_TH)
    g = O.cell_grid(p, 0, W, H, W, H)[1]

    def inside(x, y):
        return E <= x < W - E and E <= y < H - E

    def cell(x, y):
        return (y - E) // g.cell_h, (x - E) // g.cell_w

    keep = set()
    kinds = {"same_cell": 0, "cell_seam": 0, "border": 0, "tile_seam": 0}
    for (x1, y1, d1), (x2, y2, d2) in pairs:
        a, b = inside(x1, y1), inside(x2, y2)
        if a and b and cell(x1, y1) == cell(x2, y2):
            kinds["same_cell"] += 1
            if (x2 - E) // FT_W != (x1 - E) // FT_W or (y2 - E) // FT_H != (y1 - E) // FT_H:
                kinds["tile_seam"] += 1
            if abs(d1) > abs(d2):
                keep.add((x1, y1))
            elif abs(d2) > abs(d1):
                keep.add((x2, y2))
        else:
            kinds["cell_seam" if a and b else "border"] += 1
            if a:
                keep.add((x1, y1))
            if b:
                keep.add((x2, y2))
    return keep, kinds
