"""Group specs for the mixed-geometry extract entries at their limits, and a host restatement of the multi plan's layout.

Shared by test_oracle_multi_domain.py (CPU: the restatement against the oracle's level sizes, quotas and cell grids, and
each scene's facts) and test_gpu_multi_domain.py (the CUDA entries against the oracle and the single-geometry entry).
numpy only.

The restatement follows orbfe_extractor_create (level scales and quotas) and layout_geometry / build / build_multi /
begin_multi (orbfe_api.cu) in float32 where they compute in float: per geometry its level sizes, cell grids, FAST tiles,
candidate slots and kept lists, and whether the library accepts it; per call the groups' frame, FAST-work and cell-work
ranges; per plan the totals, the level-select kernel's shared memory and the group that drives each; and the capacity rule
that decides when a handle's multi plan is rebuilt.
"""
import math

import numpy as np

F32 = np.float32
EDGE = 16                   # ORBFE_EDGE
FT_W, FT_H = 120, 62        # ORBFE_FT_W x ORBFE_FT_H, the FAST kernel's tile
MAX_GROUPS = 8              # ORBFE_MULTI_MAX_GROUPS
MAX_LEVELS = 32             # ORBFE_MAX_LEVELS
MAX_FRAMES = 65535          # one grid row per frame
SMEM_DEFAULT = 48 * 1024    # dynamic shared memory a kernel gets without opting in
SMEM_LIMIT = 200 * 1024     # the plan refuses a level-select footprint past this
FAST, HARRIS = 1, 0         # score types


# ---------------------------------------------------------------------------------------------------------------------
# level tables and geometry layout
# ---------------------------------------------------------------------------------------------------------------------
def cv_round(v):
    """std::lrint on a double: round half to even"""
    return int(np.rint(np.float64(v)))


def levels(nf, sf, nl):
    """(scale, inv_scale, quota) of a handle, as orbfe_extractor_create computes them"""
    sfd = float(F32(sf))                                 # the float argument held in a double member
    scale, inv = [F32(1)], [F32(1)]
    for _ in range(1, nl):
        scale.append(F32(float(scale[-1]) * sfd))
    step = F32(1.0 / sfd)
    for _ in range(1, nl):
        inv.append(F32(inv[-1] * step))
    factor = F32(1.0 / sfd)
    nd = F32(F32(nf) * F32(F32(1) - factor)) / F32(F32(1) - F32(math.pow(float(factor), float(nl))))
    nd = F32(nd)
    quota, total = [], 0
    for _ in range(nl - 1):
        q = cv_round(nd)
        quota.append(q)
        total += q
        nd = F32(nd * factor)
    quota.append(max(nf - total, 0))
    return scale, inv, quota


class Level:
    __slots__ = ("w", "h", "quota", "cols", "rows", "cw", "ch", "ncells", "nftiles", "kept_cap", "cand")


class Layout:
    """One W x H geometry under a handle's (nf, sf, nl): its levels, or `refused` with the reason"""

    def __init__(self, nf, sf, nl, W, H):
        self.W, self.H = W, H
        self.levels, self.refused = [], None
        _, inv, quota = levels(nf, sf, nl)
        ratio = F32(F32(W) / F32(H))
        for l in range(nl):
            L = Level()
            L.w, L.h = cv_round(F32(F32(W) * inv[l])), cv_round(F32(F32(H) * inv[l]))
            L.quota = quota[l]
            if L.w < 1 or L.h < 1 or L.w > 65535 or L.h > 32767:
                self.refused = "level %d size" % l
                return
            L.cols = int(np.sqrt(F32(F32(L.quota) / F32(F32(5) * ratio)), dtype=F32))
            L.rows = int(F32(ratio * F32(L.cols)))
            Wd, Hd = L.w - 2 * EDGE, L.h - 2 * EDGE
            if L.cols < 1 or L.rows < 1:
                L.cols = L.rows = 0
                L.cw = L.ch = 1
                L.ncells = L.nftiles = 0
                L.cand = 0
            else:
                if Wd < 1 or Hd < 1:
                    self.refused = "level %d border" % l
                    return
                L.cw = int(np.ceil(F32(F32(Wd) / F32(L.cols))))
                L.ch = int(np.ceil(F32(F32(Hd) / F32(L.rows))))
                if L.cw < 2 or L.ch < 2:
                    self.refused = "level %d cells" % l
                    return
                L.ncells = L.rows * L.cols
                if (L.cols - 1) * L.cw > Wd or (L.rows - 1) * L.ch > Hd:
                    self.refused = "level %d grid" % l
                    return
                if ((FT_W + L.cw - 2) // L.cw + 1) * ((FT_H + L.ch - 2) // L.ch + 1) > 64:
                    self.refused = "level %d tile" % l
                    return
                if L.ncells > 4096 or L.cw * L.ch > (1 << 24):
                    self.refused = "level %d key layout" % l
                    return
                L.nftiles = -(-Wd // FT_W) * -(-Hd // FT_H)
                ww = np.full(L.cols, L.cw)
                ww[-1] = Wd - (L.cols - 1) * L.cw
                hh = np.full(L.rows, L.ch)
                hh[-1] = Hd - (L.rows - 1) * L.ch
                L.cand = int(np.maximum(1, ((hh[:, None] + 1) // 2) * ((ww[None, :] + 1) // 2)).sum())
            L.kept_cap = L.quota + 2 * L.ncells + 64
            self.levels.append(L)

    @property
    def ok(self):
        return self.refused is None

    @property
    def nftiles(self):
        return sum(L.nftiles for L in self.levels)

    @property
    def ncells(self):
        return sum(L.ncells for L in self.levels)

    @property
    def cand(self):
        return sum(L.cand for L in self.levels)

    @property
    def kept(self):
        return sum(L.kept_cap for L in self.levels)

    @property
    def max_kept(self):
        return max(L.kept_cap for L in self.levels)

    def partial_tiles(self):
        """level 0's detect area does not divide into whole FAST tiles"""
        return (self.W - 2 * EDGE) % FT_W != 0 and (self.H - 2 * EDGE) % FT_H != 0


def smem(max_kept, score):
    """dynamic shared memory of the level-select kernel: FAST sorts 8-byte keys in the next power of two, HARRIS holds 13
    bytes per key plus 16"""
    if score == HARRIS:
        return 13 * max_kept + 16
    n2 = 1
    while n2 < max_kept:
        n2 <<= 1
    return 8 * n2


def empty_levels(params, w, h):
    """levels whose reference cell grid is empty (ORBextractor.cc:533-547: levelCols or levelRows is 0)"""
    nf, sf, nl = params[:3]
    _, _, q = levels(nf, sf, nl)
    ratio = F32(F32(w) / F32(h))
    cols = [int(np.sqrt(F32(F32(x) / F32(F32(5) * ratio)), dtype=F32)) for x in q]
    return [l for l, c in enumerate(cols) if c < 1 or int(F32(ratio * F32(c))) < 1]


# ---------------------------------------------------------------------------------------------------------------------
# a call on the multi plan
# ---------------------------------------------------------------------------------------------------------------------
class Plan:
    """The multi plan of one call's groups [(W, H, B)] (W or H 0: an empty group) under params (nf, sf, nl, score, th).

    refused: None, or (caller's group index, reason) of the first group the plan refuses, a layout refusal or a
    level-select footprint past SMEM_LIMIT.  groups: per planned group a dict of its layout and its frame0, fwork0, cwork0
    in this call."""

    def __init__(self, params, spec):
        nf, sf, nl, score = params[:4]
        self.refused, self.groups, self.score = None, [], score
        frame = fw = cw = 0
        for g, (W, H, B) in enumerate(spec):
            if W <= 0 or H <= 0:
                continue
            lay = Layout(nf, sf, nl, W, H)
            if not lay.ok:
                self.refused = (g, lay.refused)
                return
            if smem(lay.max_kept, score) > SMEM_LIMIT:
                self.refused = (g, "level-select")
                return
            self.groups.append(dict(index=g, layout=lay, W=W, H=H, B=B, frame0=frame, fwork0=fw, cwork0=cw,
                                    nftiles=lay.nftiles, ncells=lay.ncells))
            frame += B
            fw += lay.nftiles * B
            cw += lay.ncells * B
        self.nframes, self.nfwork, self.ncwork = frame, fw, cw

    def _drive(self, key):
        vals = [key(g["layout"]) for g in self.groups]
        return max(vals), self.groups[int(np.argmax(vals))]["index"]

    @property
    def cand_total(self):
        """(slots per frame, the caller's index of the group that needs them)"""
        return self._drive(lambda L: L.cand)

    @property
    def kept_total(self):
        return self._drive(lambda L: L.kept)

    @property
    def max_kept(self):
        return self._drive(lambda L: L.max_kept)

    def smem(self, score=None):
        """(level-select bytes, the caller's index of the group that drives them)"""
        m, g = self.max_kept
        return smem(m, self.score if score is None else score), g


def capacity(calls, grow=True):
    """The capacity rule of the multi plan's build over a sequence of calls on one handle, each [(W, H, B)] (W or H 0: empty).
    A call keeps the plan when its non-empty groups' (W, H) list equals the plan's and every group fits; when only the
    frames grow, every group keeps at least its old capacity (grow=False: the rule without that).  Returns [(rebuilt, capacities after the call)]."""
    geom, cap, out = None, None, []
    for spec in calls:
        g = [(W, H) for W, H, B in spec if W > 0 and H > 0]
        want = [B for W, H, B in spec if W > 0 and H > 0]
        rebuilt = False
        if g:
            if g == geom and all(w <= c for w, c in zip(want, cap)):
                pass
            else:
                if g == geom and grow:
                    want = [max(w, c) for w, c in zip(want, cap)]
                geom, cap, rebuilt = g, want, True
        out.append((rebuilt, list(cap) if cap else []))
    return out


def first_refused(W, H, sf, nl, score, lo=1000, hi=20000):
    """the smallest nfeatures from lo at which W x H lays out and the plan refuses it for its level-select footprint (some
    counts are refused earlier because their cell grid does not tile the detect area)"""
    for nf in range(lo, hi):
        lay = Layout(nf, sf, nl, W, H)
        if lay.ok and smem(lay.max_kept, score) > SMEM_LIMIT:
            return nf
    raise AssertionError("no refusal below %d" % hi)


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
# partners of a domain scene's group: one larger, one portrait, valid under every scene's handle parameters
PARTNERS = [(1280, 720), (480, 640)]
DOMAIN_PARAMS = [(800, 1.2, 3), (500, 1.2, 1), (1500, 1.2, 1), (1500, 1.2, 2), (1500, 1.2, 3), (2000, 1.2, 8)]
POSITIONS = ("first", "middle", "last")


def placed(scene, partners, pos):
    """the scene's groups (a list) first, between the partners, or last"""
    return {"first": scene + partners, "middle": partners[:1] + scene + partners[1:], "last": partners + scene}[pos]


# a geometry with no FAST tile and no cell at any level: 200 x 1200 at nf 100 over 8 levels (levelRows = 0 everywhere)
TILELESS = (200, 1200)
TILELESS_PARAMS = (100, 1.2, 8, FAST, 20)
TILELESS_PARTNERS = [(640, 480), (1280, 720), (480, 640)]
# the tile-less group first, in the middle, last and twice in a row among groups with tiles: [(W, H, B)]
TILELESS_CALLS = {
    "first": [(200, 1200, 2), (640, 480, 1), (1280, 720, 1)],
    "middle": [(640, 480, 1), (200, 1200, 1), (480, 640, 2)],
    "last": [(1280, 720, 1), (480, 640, 1), (200, 1200, 2)],
    "twice": [(640, 480, 2), (200, 1200, 1), (200, 1200, 2), (1280, 720, 1)],
}

# eight distinct geometries, the group limit: landscape, portrait, odd and partial last FAST tiles
EIGHT = [(1280, 720), (640, 480), (480, 640), (752, 480), (1241, 376), (1001, 333), (800, 600), (544, 960)]
EIGHT_BATCH = [1, 2, 1, 1, 1, 1, 1, 2]
EIGHT_SETTINGS = {   # (levels, scale): 8 x 32 fills the level table; 2.0 and 3.0 take the generic resize path
    "8x1.2": (8, 1.2), "16x1.05": (16, 1.05), "32x1.01": (32, 1.01), "3x2.0": (3, 2.0), "2x3.0": (2, 3.0)}
EIGHT_NF = 1000

# the level-select kernel past 48 KB in a multi plan (one level)
SMEM_SETS = {"fast": ((7000, 1.2, 1, FAST, 10), [(1600, 1200, 1), (1280, 800, 1), (752, 480, 1)]),
             "harris": ((5000, 1.2, 1, HARRIS, 10), [(1600, 1200, 1), (960, 540, 1), (768, 1024, 1)])}
# a single-geometry plan needing less than SMEM_SETS but more than 48 KB: the attribute must not drop back to it
SMEM_SMALLER = {"fast": ((5000, 1.2, 1, FAST, 10), (1024, 768)), "harris": ((3000, 1.2, 1, HARRIS, 10), (640, 480))}

# geometry pairs whose level-select footprints split at one nfeatures (one level, scale 1.2): the first geometry runs
# there, the second is refused
REFUSAL_PAIRS = {"fast": (FAST, 11713, (1280, 800), (1440, 800)),
                 "harris": (HARRIS, 11261, (1920, 1080), (1600, 1200))}

# capacity sequences on one handle: frames per group of CAP_GEOMS, and the plan builds after each call
CAP_GEOMS = [(640, 480), (1280, 720), (480, 640)]
CAP_SEQUENCE = [(1, 1, 1), (3, 1, 1), (1, 1, 1), (3, 1, 4), (3, 1, 4), (1, 1, 5), (3, 1, 5), (2, 1, 2)]
CAP_BUILDS = [1, 2, 2, 3, 3, 4, 4, 4]
CAP_MAX = (3, 1, 5)          # frames each group's caller buffer holds

# 65535 frames, the grid-row limit, across two small groups (one cell, one FAST tile each)
LIMIT_PARAMS = (19, 1.2, 1, FAST, 20)
LIMIT_GROUPS = [(64, 64, 32768), (80, 48, 32767)]
LIMIT_DISTINCT = 7           # distinct frames tiled through each group


def spec_of(geoms, batch):
    return [(W, H, B) for (W, H), B in zip(geoms, batch)]
