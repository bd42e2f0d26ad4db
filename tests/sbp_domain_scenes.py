"""Constructed scenes for the accept logic of the fused projection matcher (sbp_device_kernel in
orb_slam_b200/csrc/match_kernels.cu), numpy only.

The kernel computes the reference's sequential accept loop (ORBmatcher.cc) with three parallel mechanisms the reference
does not have: deferred acceptance for the best-only rule (rule 0), reservation rounds with a sequential warp after
SBP_MAX_ROUNDS for the second-best rules (1, 2), and one sequential warp with a prefetch of the next list for
SearchForInitialization (MODE 2).  Random content decides almost every query in the first round, so these scenes build the
contention on purpose: reservation chains past the 48-round fallback, displacement cascades, MODE-2 re-assignment, and
rotation histograms on their boundaries.

Every scene is plain arrays: a frame of slots (keypoints and descriptors), explicit query windows with descriptors, the
slots occupied on entry, and the candidate list each window is designed to hold.  Distances come from explicit bit flips
(`mask`), so "q is 10 from s" holds exactly.  Keypoints sit on rows 40 px apart (one grid-cell row each) with 10 px
between chain slots, so a 6 px window holds exactly its designed list; `lists_of` checks that against GetFeaturesInArea.

`sequential` is the plain-Python accept loop written from ORBmatcher.cc (rules 0-2, the MODE-2 rule, the rotation histogram
and ComputeThreeMaxima); it is the reference the oracle and the kernel are held to.  `rounds` and `passes` model the kernel's
schedule: the round in which each rule-1/2 query decides and which queries remain for the warp after 48 rounds, and the
number of synchronous deferred-acceptance passes of rule 0.  `VARIANTS` are wrong versions of the loop; each scene names
the variants its outcome must change under.
"""
import copy

import numpy as np

from bow_domain_scenes import mask

W, H = 2560, 1920            # 64 x 48 grid cells of 40 x 40 px
TH_HIGH, TH_LOW = 100, 50
MAX_ROUNDS = 48              # SBP_MAX_ROUNDS
INT_MAX = 2 ** 31 - 1
R = 6.0                      # window radius: the slots 5 px away are in, the ones 15 px away are out
F32 = np.float32

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])

VARIANTS = ("simultaneous", "fallback_reruns_decided", "fallback_drops_undecided", "pick_only_commit", "last_min_wins",
            "th_exclusive", "ratio_strict", "level_ignored", "stale_prefetched_distance", "three_maxima_le", "rot_le_zero_wrap")


# ---------------------------------------------------------------------------------------------------------------------
# scene construction

class Scene:
    """kps / desc: the searched frame (slots); q*: the query windows; occ: slots occupied on entry (bool); lists: the
    designed candidate list of every query (slot indices in GetFeaturesInArea order); dist[q]: distances in list order."""

    def __init__(self, name, rule, nnratio=0.75, th_dist=TH_HIGH, hist=0, changes=(), facts=None):
        self.name, self.rule, self.nnratio, self.th_dist, self.hist = name, rule, nnratio, th_dist, hist
        self.changes = tuple(changes)
        self.facts = dict(facts or {})

    @property
    def nq(self):
        return len(self.qu)

    @property
    def n(self):
        return len(self.kps)

    def slot_owner(self):
        so = np.full(self.n, -1, np.int32)
        so[self.occ] = 1 << 20    # an owner no query index of any scene reaches
        return so


class Builder:
    """Slots, queries and the distances between them.  Queries created with `like=` share the descriptor of an earlier
    query.  The (query descriptor, slot) distance graph must be a forest: the descriptors are laid out by walking it."""

    def __init__(self, seed=0):
        self.rng = np.random.default_rng(seed)
        self.sx, self.sy, self.soct, self.sang = [], [], [], []
        self.qu, self.qv, self.qr, self.qlo, self.qhi, self.qang, self.qrep = [], [], [], [], [], [], []
        self.lists, self.dists = [], []
        self.occ = []
        self.row = 0

    def next_row(self):
        y = 20.0 + 40.0 * self.row
        self.row += 1
        assert y < H
        return y

    def slot(self, x, y, octave=0, angle=0.0, occupied=False):
        assert 0 <= x < W and 0 <= y < H
        self.sx.append(x); self.sy.append(y); self.soct.append(octave); self.sang.append(angle)
        if occupied:
            self.occ.append(len(self.sx) - 1)
        return len(self.sx) - 1

    def query(self, u, v, cands, r=R, lo=-1, hi=-1, angle=0.0, like=None):
        """cands: [(slot, distance)] in the designed list order."""
        self.qu.append(u); self.qv.append(v); self.qr.append(r); self.qlo.append(lo); self.qhi.append(hi); self.qang.append(angle)
        self.qrep.append(len(self.qu) - 1 if like is None else self.qrep[like])
        self.lists.append([s for s, _ in cands])
        self.dists.append([d for _, d in cands])
        return len(self.qu) - 1

    def build(self, scene):
        n, nq = len(self.sx), len(self.qu)
        kps = np.zeros(n, KP_DTYPE)
        kps["x"], kps["y"], kps["octave"], kps["angle"] = self.sx, self.sy, self.soct, self.sang
        kps["size"], kps["response"], kps["class_id"] = 31.0, 1.0, -1
        # descriptors: walk the forest of (query representative, slot) distance edges
        adj = {}
        for q in range(nq):
            a = ("q", self.qrep[q])
            for s, d in zip(self.lists[q], self.dists[q]):
                b = ("s", s)
                adj.setdefault(a, {}); adj.setdefault(b, {})
                if b in adj[a]:
                    assert adj[a][b] == d, "one query descriptor with two distances to one slot"
                adj[a][b] = d; adj[b][a] = d
        desc_of = {}
        nodes = [("s", s) for s in range(n)] + [("q", q) for q in sorted(set(self.qrep))]
        for root in nodes:
            if root in desc_of:
                continue
            desc_of[root] = self.rng.integers(0, 256, 32, dtype=np.uint8)
            stack, parent = [root], {root: None}
            while stack:
                a = stack.pop()
                for b, d in adj.get(a, {}).items():
                    if b == parent[a]:
                        continue
                    assert b not in desc_of, "the distance graph has a cycle"
                    desc_of[b] = desc_of[a] ^ mask(self.rng.choice(256, d, replace=False))
                    parent[b] = a
                    stack.append(b)
        scene.kps = kps
        scene.desc = np.stack([desc_of[("s", s)] for s in range(n)]) if n else np.zeros((0, 32), np.uint8)
        scene.qdesc = np.stack([desc_of[("q", self.qrep[q])] for q in range(nq)])
        scene.qu, scene.qv, scene.qr = (np.asarray(a, np.float32) for a in (self.qu, self.qv, self.qr))
        scene.qlo, scene.qhi = np.asarray(self.qlo, np.int32), np.asarray(self.qhi, np.int32)
        scene.qangle = np.asarray(self.qang, np.float32)
        scene.occ = np.zeros(n, bool)
        scene.occ[self.occ] = True
        scene.lists = [list(l) for l in self.lists]
        scene.dist = [list(d) for d in self.dists]
        return scene


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


def check_distances(sc):
    """The distances in the scene are the designed ones."""
    for q in range(sc.nq):
        for s, d in zip(sc.lists[q], sc.dist[q]):
            assert hamming(sc.qdesc[q], sc.desc[s]) == d, (sc.name, q, s, d)


def lists_of(sc, oracle_frame):
    """GetFeaturesInArea of every query window (the candidate lists the matcher enumerates)."""
    return [list(oracle_frame.features_in_area(float(sc.qu[q]), float(sc.qv[q]), float(sc.qr[q]), int(sc.qlo[q]), int(sc.qhi[q])))
            for q in range(sc.nq)]


# ---------------------------------------------------------------------------------------------------------------------
# rules 1 and 2: reservation chains

def _tail(b, y, x, s_prev, L, rule, ties=False):
    """The last query of a chain: its list is the chain's last slot `s_prev` followed by L - 1 private fillers (all at one
    point, so in index order).  L = 1: only s_prev at 10, accepted without a second.  Otherwise the best is in the list's
    last 32-lane chunk (rule 1: position L - 1; rule 2: positions 31 and 32 tied at 20 on octaves 0 and 1 when L > 32, else
    position L - 1 at 20 with the second at L - 2 on another octave and above the ratio).  `ties` (rule 1, L > 32):
    positions 31 and 32 tied at 20 instead, so the best and the second are equal and the first of them is the match."""
    if L == 1:
        return b.query(x, y, [(s_prev, 10)])
    cands = [(s_prev, 30)]
    fx = b.sx[s_prev] + 3.0
    for p in range(1, L):
        d, o = 40, 0
        if rule == 1 and (p in (31, 32) if ties else p == L - 1):
            d = 20
        if rule == 2:
            if L > 32 and p in (31, 32):
                d, o = 20, p - 31
            elif L <= 32 and p == L - 1:
                d = 20
            elif L <= 32 and L >= 3 and p == L - 2:
                d, o = 22, 1
        cands.append((b.slot(fx, y, octave=o), d))
    return b.query(x, y, cands)


def add_chain(b, depth, blocked, rule, tail=2, dist=(10, 12), ties=False):
    """q_i lists s_i at 10 and s_(i+1) at 12 (both octave 0).  nnratio 0.75: with both slots free q_i rejects (10 > 9);
    with s_i taken it takes s_(i+1).  s_0 occupied on entry: every query shifts by one; s_0 free: every query rejects, and q_i
    decides in round i + 1.  `dist` replaces (10, 12); `tail` = the last query's list length and `ties` its tie (see _tail).
    Returns the chain's query indices."""
    y = b.next_row()
    x0 = 10.0
    slots = [b.slot(x0, y, occupied=blocked)]
    qs = []
    for i in range(depth):
        last = i == depth - 1
        xc = x0 + 10.0 * i + 5.0
        if last and tail != 2:
            qs.append(_tail(b, y, xc, slots[i], tail, rule, ties))
        else:
            slots.append(b.slot(x0 + 10.0 * (i + 1), y))
            qs.append(b.query(xc, y, [(slots[i], dist[0]), (slots[i + 1], dist[1])]))
    return qs


def add_rerun_pair(b):
    """R lists a at 10 and b at 12 (rejects: both free); X > R lists b alone at 10 (accepts).  R decides in round 1 and X
    in round 2.  Re-run after the rounds, R would find a alone and accept it."""
    y = b.next_row()
    a, s = b.slot(100.0, y), b.slot(110.0, y)
    r = b.query(105.0, y, [(a, 10), (s, 12)])
    x = b.query(115.0, y, [(s, 10)])
    return r, x


def add_pick_only_pair(b):
    """P0 lists a alone at 10 (accepts).  P1 lists a at 12 and b at 10: b is P1's pick and carries only P1's stamp in round
    1, but a carries P0's.  Sequentially P1 sees b alone and accepts; deciding on the pick alone it sees a and b (10 > 9)."""
    y = b.next_row()
    a, s = b.slot(300.0, y), b.slot(310.0, y)
    p0 = b.query(295.0, y, [(a, 10)])
    p1 = b.query(305.0, y, [(a, 12), (s, 10)])
    return p0, p1


def add_ratio_edges(b, rule):
    """Single queries on the rule's comparisons: rule 1 at 9 vs 12 (== 0.75 * 12, accepted) and 10 vs 12 (rejected); rule 2
    at 9 vs 12 on one octave (accepted), 10 vs 12 on one octave (rejected), 10 vs 12 on two octaves (accepted)."""
    y = b.next_row()
    out = []
    x = 500.0
    cases = [(9, 12, 0), (10, 12, 0)] + ([(10, 12, 1)] if rule == 2 else [])
    for d1, d2, o2 in cases:
        a, s = b.slot(x, y), b.slot(x + 10.0, y, octave=o2)
        out.append(b.query(x + 5.0, y, [(a, d1), (s, d2)]))
        x += 40.0
    # TH_HIGH: best 100 kept, 101 dropped (no second)
    for d in (100, 101):
        out.append(b.query(x + 5.0, y, [(b.slot(x, y), d)]))
        x += 40.0
    return out


def chains_scene(rule, depths=(1, 47, 48, 49, 50, 200), seed=1):
    """Free and blocked chains of every depth, then a re-run pair, a pick-only pair and the ratio edges, in one job."""
    b = Builder(seed)
    sc = Scene("chains-rule%d" % rule, rule)
    sc.facts["free"] = {d: add_chain(b, d, False, rule) for d in depths}
    sc.facts["blocked"] = {d: add_chain(b, d, True, rule) for d in depths}
    sc.facts["rerun"] = add_rerun_pair(b)
    sc.facts["pick_only"] = add_pick_only_pair(b)
    sc.facts["edges"] = add_ratio_edges(b, rule)
    sc.changes = ("simultaneous", "fallback_reruns_decided", "fallback_drops_undecided", "pick_only_commit", "th_exclusive",
                  "ratio_strict") + (("level_ignored",) if rule == 2 else ())
    return b.build(sc)


def tails_scene(rule, lengths=(1, 31, 32, 33, 64, 65), seed=2):
    """Free 49-deep chains whose last query, the first one the rounds leave to the warp, lists 1-65 entries; the warp's
    reductions cross 32-lane chunks.  Rule 2 puts ties for best and second at positions 31 / 32."""
    b = Builder(seed)
    sc = Scene("tails-rule%d" % rule, rule)
    sc.facts["tails"] = {L: add_chain(b, 49, False, rule, tail=L)[-1] for L in lengths}
    sc.changes = ("fallback_drops_undecided",) + (("last_min_wins",) if rule == 2 else ())
    return b.build(sc)


def tie_tails_scene(lengths=(33, 64, 65), seed=8):
    """Rule 1 with nnratio 1.0, where a tie for best passes the ratio test (20 <= 20): free 49-deep chains whose queries
    list two slots at 101 (above TH_HIGH, so every chain query rejects, one round after the previous one), ending in a warp
    query with the best tied at positions 31 / 32.  The first of the tie is the match; the last minimum would take 32."""
    b = Builder(seed)
    sc = Scene("ties-rule1", 1, nnratio=1.0)
    sc.facts["tails"] = {L: add_chain(b, 49, False, 1, tail=L, dist=(101, 101), ties=True)[-1] for L in lengths}
    sc.changes = ("fallback_drops_undecided", "last_min_wins")
    return b.build(sc)


# ---------------------------------------------------------------------------------------------------------------------
# rule 0: displacement cascades

def star_scene(K, d=20, seed=3, th_dist=TH_HIGH):
    """K queries with one descriptor share the same K slots (one point, so the list is the slot order), every slot at d:
    the ranking is the list position.  Query q ends on slot q, after K deferred-acceptance passes."""
    b = Builder(seed)
    y = b.next_row()
    slots = [b.slot(100.0, y) for _ in range(K)]
    q0 = None
    for q in range(K):
        qq = b.query(100.0, y, [(s, d) for s in slots], like=q0)
        q0 = qq if q0 is None else q0
    sc = Scene("star-%d" % K, 0, th_dist=th_dist, changes=("simultaneous", "last_min_wins"))
    sc.facts["K"] = K
    return b.build(sc)


def add_ladder(b, depth, occupied_at=()):
    """q_i lists s_i and s_(i+1), both at 15 (tie: list position decides).  s_0 occupied: each query displaces the next;
    `occupied_at`: slots occupied on entry inside the cascade (the query before it gets nothing, the one at it shifts on)."""
    y = b.next_row()
    slots = [b.slot(10.0, y, occupied=True)]
    qs = []
    for i in range(depth):
        slots.append(b.slot(10.0 + 10.0 * (i + 1), y, occupied=(i + 1) in occupied_at))
        qs.append(b.query(15.0 + 10.0 * i, y, [(slots[i], 15), (slots[i + 1], 15)]))
    return qs


def ladder_scene(depths=(1, 48, 49, 200), seed=4, th_dist=TH_HIGH):
    b = Builder(seed)
    sc = Scene("ladders", 0, th_dist=th_dist)
    sc.facts["ladders"] = {d: add_ladder(b, d) for d in depths}
    sc.facts["holed"] = add_ladder(b, 60, occupied_at=(20, 40))
    y = b.next_row()
    sc.facts["th"] = [b.query(105.0 + 40 * i, y, [(b.slot(100.0 + 40 * i, y), th_dist + i)]) for i in range(2)]  # kept, dropped
    sc.changes = ("simultaneous", "th_exclusive")
    return b.build(sc)


# ---------------------------------------------------------------------------------------------------------------------
# MODE 2 (SearchForInitialization): re-assignment.  Every query is a level-0 F1 feature; the window is R for all of them.

def init_scene(seed=5):
    b = Builder(seed)
    sc = Scene("init", 3, nnratio=0.75, th_dist=TH_LOW, hist=1)
    y = b.next_row()
    # prefetch: q takes s at 20; for q + 1 (the next query with work, same ballot group) s is at 25 and t at 40
    s, t = b.slot(100.0, y), b.slot(110.0, y)
    q = b.query(95.0, y, [(s, 20)])
    b.query(105.0, y, [(s, 25), (t, 40)])
    sc.facts["prefetch"] = (q, s, t)
    # re-assignment chain on one slot: 30, then 20, then 10.  The displaced features keep their histogram entries (bin 5:
    # angle difference 150), and with them bin 5 keeps a live match (p) against 21 matches in bin 0.
    y = b.next_row()
    s = b.slot(300.0, y)
    chain = [b.query(300.0, y, [(s, d)], angle=150.0 if d > 10 else 0.0) for d in (30, 20, 10)]
    p = b.query(345.0, y, [(b.slot(340.0, y), 5)], angle=150.0)
    sc.facts["reassign"] = (chain, s, p)
    y = b.next_row()
    sc.facts["bin0"] = [b.query(505.0 + 20 * i, y, [(b.slot(500.0 + 20 * i, y), 5)]) for i in range(20)]
    # lists of 32 and 40 entries (one point): the best at position 31 / 35 at 20, the rest at 45
    y = b.next_row()
    lq = []
    for k, (L, best) in enumerate(((32, 31), (40, 35))):
        x = 100.0 + 100 * k
        cands = [(b.slot(x, y), 20 if p == best else 45) for p in range(L)]
        lq.append(b.query(x, y, cands))
    sc.facts["long"] = lq
    # TH_LOW: 50 kept, 51 dropped; the strict ratio test: 9 vs 12 (== 0.75 * 12) dropped, 8 vs 12 kept
    y = b.next_row()
    sc.facts["th"] = [b.query(105.0 + 40 * i, y, [(b.slot(100.0 + 40 * i, y), d)]) for i, d in enumerate((50, 51))]
    rq = []
    for i, d1 in enumerate((9, 8)):
        x = 300.0 + 40 * i
        rq.append(b.query(x + 5.0, y, [(b.slot(x, y), d1), (b.slot(x + 10.0, y), 12)]))
    sc.facts["ratio"] = rq
    sc.changes = ("stale_prefetched_distance", "th_exclusive", "ratio_strict")
    return b.build(sc)


# ---------------------------------------------------------------------------------------------------------------------
# rotation histogram (rule 0, independent single-candidate queries; angle = query angle - slot angle)

def rot_bin(a1, a2, variant=None):
    """round((a1 - a2 [+360]) * (1.0f/30)) in float32, half away from zero; 30 -> 0."""
    rot = F32(F32(a1) - F32(a2))
    if rot < 0 or (variant == "rot_le_zero_wrap" and rot <= 0):
        rot = F32(rot + F32(360.0))
    x = float(F32(rot * (F32(1.0) / F32(30))))
    b = int(np.floor(abs(x) + 0.5)) * (1 if x >= 0 else -1)
    return 0 if b == 30 else b


def half_bin_below():
    """The largest float32 angle difference that rounds to bin 0 (rot * (1.0f/30) < 0.5), and the next one up (bin 1)."""
    r = F32(15.0)
    while F32(r * (F32(1.0) / F32(30))) >= F32(0.5):
        r = np.nextafter(r, F32(0))
    return float(r), float(np.nextafter(r, F32(100)))


def hist_scene(counts, seed=6, name=None):
    """counts: [((a_query, a_slot), number of matches)] (a list: -0.0 and 0.0 are one dict key); each match is one query
    with one private slot at distance 5."""
    b = Builder(seed)
    sc = Scene(name or "hist", 0, hist=1)
    y = b.next_row()
    x = 10.0
    groups = {}
    for (aq, as_), c in counts:
        for _ in range(c):
            if x > W - 20:
                y, x = b.next_row(), 10.0
            groups.setdefault((repr(aq), as_), []).append(b.query(x + 5.0, y, [(b.slot(x, y, angle=as_), 5)], angle=aq))
            x += 20.0
    sc.facts["groups"] = groups
    return b.build(sc)


def hist_scenes():
    lo, hi = half_bin_below()
    tiny = float(np.nextafter(F32(0), F32(1)))
    out = []
    # max2 == 0.1f * max1 (kept) and max3 == 0.1f * max1 (kept); one below (dropped)
    out.append(hist_scene([((0.0, 0.0), 10), ((90.0, 0.0), 1)], name="max2-at"))
    out.append(hist_scene([((0.0, 0.0), 20), ((90.0, 0.0), 2), ((180.0, 0.0), 2)], name="max3-at"))
    out.append(hist_scene([((0.0, 0.0), 20), ((90.0, 0.0), 1), ((180.0, 0.0), 1)], name="max2-below"))
    out.append(hist_scene([((0.0, 0.0), 20), ((90.0, 0.0), 2), ((180.0, 0.0), 1)], name="max3-below"))
    # ties for the first maximum: four bins of 5, the first three kept
    out.append(hist_scene([((0.0, 0.0), 5), ((120.0, 0.0), 5), ((210.0, 0.0), 5), ((270.0, 0.0), 5)], name="max-ties"))
    # angle differences: +0 and -0.0 (bin 0), just below 0 (wraps to 360: bin 12), the half-bin (bins 0 / 1); bin 0 holds
    # 10 only when the zero differences count there, so the wrap variant moves the maxima
    out.append(hist_scene([((0.0, 0.0), 4), ((-0.0, 0.0), 4), ((-tiny, 0.0), 9), ((lo, 0.0), 1), ((hi, 0.0), 9),
                           ((200.0, 0.0), 2), ((330.0, 0.0), 1)], name="angles"))
    for sc in out:
        sc.changes = ("three_maxima_le",) if sc.name in ("max2-at", "max3-at") else ()
    out[-1].changes = ("rot_le_zero_wrap",)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the sequential model (ORBmatcher.cc): rules 0-2 over explicit candidate lists, the MODE-2 rule, histogram, three maxima

def _best_second(cands, usable, octave, variant):
    """The strict-< best / second update of the reference's loops (:1558-1570, :451-466, :94-110): first minimum wins."""
    b1, b2, i1, l1, l2 = INT_MAX, INT_MAX, -1, -1, -1
    lt = (lambda a, c: a <= c) if variant == "last_min_wins" else (lambda a, c: a < c)
    for s, d in cands:
        if not usable(s, d):
            continue
        if lt(d, b1):
            b2, l2, b1, i1, l1 = b1, l1, d, s, octave[s]
        elif lt(d, b2):
            b2, l2 = d, octave[s]
    return b1, b2, i1, l1, l2


def accept(rule, b1, b2, l1, l2, nnratio, th_dist, variant=None):
    le = (lambda a, c: a < c) if variant == "th_exclusive" else (lambda a, c: a <= c)
    r = F32(nnratio)
    if rule == 0:
        return b1 != INT_MAX and le(b1, th_dist)
    if rule == 1:   # (float)best <= (float)second * nnratio && best <= TH_HIGH
        rt = F32(b1) < F32(F32(b2) * r) if variant == "ratio_strict" else F32(b1) <= F32(F32(b2) * r)
        return bool(rt) and le(b1, TH_HIGH)
    if rule == 2:   # best <= TH_HIGH && !(bestLevel == bestLevel2 && best > nnratio * second)
        same = l1 == l2 or variant == "level_ignored"
        worse = F32(b1) >= F32(r * F32(b2)) if variant == "ratio_strict" else F32(b1) > F32(r * F32(b2))
        return le(b1, TH_HIGH) and not (same and bool(worse))
    # MODE 2: best <= TH_LOW && (float)best < (float)second * nnratio
    rt = F32(b1) <= F32(F32(b2) * r) if variant == "ratio_strict" else F32(b1) < F32(F32(b2) * r)
    return b1 != INT_MAX and le(b1, TH_LOW) and bool(rt)


def three_maxima(counts, variant=None):
    m1 = m2 = m3 = 0
    i1 = i2 = i3 = -1
    for i, s in enumerate(counts):
        if s > m1:
            m3, m2, m1, i3, i2, i1 = m2, m1, s, i2, i1, i
        elif s > m2:
            m3, m2, i3, i2 = m2, s, i2, i
        elif s > m3:
            m3, i3 = s, i
    lt = (lambda a, c: a <= c) if variant == "three_maxima_le" else (lambda a, c: a < c)
    t = F32(F32(0.1) * F32(m1))
    if lt(F32(m2), t):
        i2 = i3 = -1
    elif lt(F32(m3), t):
        i3 = -1
    return i1, i2, i3


def _cands(sc, q):
    return list(zip(sc.lists[q], sc.dist[q]))


def _hist_filter(sc, owner, entries, variant, counts_out=None):
    """entries: [(query, slot)] in accept order; removes the matches outside the three maxima."""
    counts = [0] * 30
    bins = []
    for q, s in entries:
        bn = rot_bin(sc.qangle[q], sc.kps["angle"][s], variant)
        counts[bn] += 1
        bins.append(bn)
    keep = three_maxima(counts, variant)
    if counts_out is not None:
        counts_out.extend(counts)
    return [(q, s) for (q, s), bn in zip(entries, bins) if bn not in keep]


def sequential(sc, variant=None, decide_at=None):
    """The reference's loop.  Returns (nmatches, slot_owner): slot_owner[s] = query index for matches of this call, the
    scene's occupied marker for slots occupied on entry, -1 otherwise.  MODE 2 (rule 3) returns (nmatches, match12).
    `decide_at`: per query the free set to decide against instead of the current one (used by the schedule variants)."""
    if sc.rule == 3:
        return _sequential_init(sc, variant)
    so = sc.slot_owner()
    octave = sc.kps["octave"]
    entries = []
    snapshot = so.copy()
    for q in range(sc.nq):
        ref = snapshot if variant == "simultaneous" else so
        b1, b2, i1, l1, l2 = _best_second(_cands(sc, q), lambda s, d: ref[s] < 0, octave, variant)
        if not accept(sc.rule, b1, b2, l1, l2, sc.nnratio, sc.th_dist, variant):
            continue
        if so[i1] >= 0:      # simultaneous: a lower query already took it
            continue
        so[i1] = q
        entries.append((q, i1))
    if sc.hist == 1:
        for q, s in _hist_filter(sc, so, entries, variant):
            so[s] = -1
    return int((so >= 0).sum() - sc.occ.sum()), so


def _sequential_init(sc, variant=None):
    """SearchForInitialization (:598-713): a slot is re-assigned to a later query that is strictly closer; every accepted
    query keeps its histogram entry; the three-maxima filter unmatches only queries that are still matched."""
    n1 = sc.nq
    mdist = [INT_MAX] * sc.n
    m21 = [-1] * sc.n
    m12 = np.full(n1, -1, np.int32)
    entries = []
    before = list(mdist)          # vMatchedDistance before the previous query with work
    for q in range(n1):
        cands = _cands(sc, q)
        if not cands:
            continue
        md = before if variant == "stale_prefetched_distance" else mdist
        before = list(mdist)
        b1, b2, i1, _, _ = _best_second(cands, lambda s, d: md[s] > d, sc.kps["octave"], variant)
        if not accept(3, b1, b2, 0, 0, sc.nnratio, TH_LOW, variant):
            continue
        if m21[i1] >= 0:
            m12[m21[i1]] = -1
        m12[q], m21[i1], mdist[i1] = i1, q, b1
        entries.append((q, i1))
    if sc.hist == 1:
        for q, s in _hist_filter(sc, None, entries, variant):
            m12[q] = -1
    return int((m12 >= 0).sum()), m12


def hist_counts(sc):
    """The 30 bin counts of the call's histogram on the sequential model (MODE 2: every accepted query, displaced or not)."""
    if sc.rule == 3:
        mdist, m21, entries = [INT_MAX] * sc.n, [-1] * sc.n, []
        for q in range(sc.nq):
            cands = _cands(sc, q)
            b1, b2, i1, _, _ = _best_second(cands, lambda s, d: mdist[s] > d, sc.kps["octave"], None)
            if cands and accept(3, b1, b2, 0, 0, sc.nnratio, TH_LOW):
                m21[i1], mdist[i1] = q, b1
                entries.append((q, i1))
    else:
        h = copy.copy(sc)
        h.hist = 0
        _, so = sequential(h)
        entries = sorted((int(so[s]), s) for s in range(sc.n) if so[s] >= 0 and not sc.occ[s])
    counts = []
    _hist_filter(sc, None, entries, None, counts)
    return counts


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's schedule

def rounds(sc, variant=None, max_rounds=MAX_ROUNDS):
    """Rules 1/2: the reservation rounds followed by the sequential warp.  Every undecided query stamps every free slot of
    its list; it decides (accept or reject) when its stamp survived on all of them ('pick_only_commit': on its pick).  A
    round's takes are visible from the next round on.  Returns (nmatches, slot_owner, decided_round, warp_queries): the
    round each query decided in (0 = no candidates) and the queries left to the warp, in the order it takes them."""
    assert sc.rule in (1, 2)
    so = sc.slot_owner()
    octave = sc.kps["octave"]
    undecided = [q for q in range(sc.nq) if sc.lists[q]]
    rnd = {q: 0 for q in range(sc.nq) if not sc.lists[q]}
    entries = []
    for r in range(1, max_rounds + 1):
        if not undecided:
            break
        stamp, free = {}, {}
        for q in undecided:
            free[q] = [s for s in sc.lists[q] if so[s] < 0]
            for s in free[q]:
                stamp[s] = min(stamp.get(s, q), q)
        takes, left = [], []
        for q in undecided:
            if not free[q]:
                rnd[q] = r
                continue
            b1, b2, i1, l1, l2 = _best_second(_cands(sc, q), lambda s, d: so[s] < 0, octave, None)
            own = [stamp[i1] == q] if variant == "pick_only_commit" else [stamp[s] == q for s in free[q]]
            if not all(own):
                left.append(q)
                continue
            rnd[q] = r
            if accept(sc.rule, b1, b2, l1, l2, sc.nnratio, sc.th_dist, variant):
                takes.append((q, i1))
        for q, s in takes:
            so[s] = q
            entries.append((q, s))
        undecided = left
    if variant == "fallback_drops_undecided":
        warp = []
    elif variant == "fallback_reruns_decided":
        warp = [q for q in range(sc.nq) if sc.lists[q]] if undecided else []
    else:
        warp = list(undecided)
    for q in warp:
        b1, b2, i1, l1, l2 = _best_second(_cands(sc, q), lambda s, d: so[s] < 0, octave, None)
        if accept(sc.rule, b1, b2, l1, l2, sc.nnratio, sc.th_dist, variant):
            so[i1] = q
            entries.append((q, i1))
    if sc.hist == 1:
        for q, s in _hist_filter(sc, so, sorted(entries), None):
            so[s] = -1
    return int((so >= 0).sum() - sc.occ.sum()), so, rnd, list(undecided)


def passes(sc):
    """Rule 0: deferred acceptance in synchronous passes (every query reads the holders as they were at the start of the
    pass).  A query proposes to its best slot (distance, then list position, within th_dist) that no lower query holds; the
    lowest proposer holds a slot.  Returns (nmatches, slot_owner, number of passes including the last one that changes
    nothing)."""
    assert sc.rule == 0
    BIG = 1 << 40
    holder = np.where(sc.occ, -1, BIG).astype(np.int64)
    pos = {q: None for q in range(sc.nq)}   # None = not started, -1 = exhausted
    keys = [sorted((d, p, s) for p, (s, d) in enumerate(_cands(sc, q)) if d <= sc.th_dist) for q in range(sc.nq)]
    npass = 0
    while True:
        npass += 1
        snap = holder.copy()
        changed = False
        for q in range(sc.nq):
            k = pos[q]
            if k == -1:
                continue
            if k is not None and snap[keys[q][k][2]] == q:
                continue
            if k is not None and snap[keys[q][k][2]] > q:
                holder[keys[q][k][2]] = min(holder[keys[q][k][2]], q)
                changed = True
                continue
            start = 0 if k is None else k + 1
            nxt = next((j for j in range(start, len(keys[q])) if snap[keys[q][j][2]] > q), -1)
            pos[q] = nxt
            changed = True
            if nxt != -1:
                holder[keys[q][nxt][2]] = min(holder[keys[q][nxt][2]], q)
        if not changed:
            break
    so = sc.slot_owner()
    entries = []
    for q in range(sc.nq):
        if pos[q] not in (None, -1) and holder[keys[q][pos[q]][2]] == q:
            so[keys[q][pos[q]][2]] = q
            entries.append((q, keys[q][pos[q]][2]))
    if sc.hist == 1:
        for q, s in _hist_filter(sc, so, entries, None):
            so[s] = -1
    return int((so >= 0).sum() - sc.occ.sum()), so, npass


def outcome(sc, variant=None):
    """The scene's outcome under a variant: the schedule variants act on the schedule model, the others on the loop."""
    if variant in ("fallback_reruns_decided", "fallback_drops_undecided", "pick_only_commit"):
        n, so, _, _ = rounds(sc, variant)
        return n, so
    return sequential(sc, variant)


# ---------------------------------------------------------------------------------------------------------------------
# launch geometry of the host guided entry: copies of orbfe::sbp_smem_fixed_bytes (match_kernels.cu) and sbp_fit_qcap
# (orbfe_api.cu, 220 KB of shared memory less 16 KB of entries).  test_gpu_sbp_domain.py checks the launch count they
# predict against the matcher's launch counter.

def sbp_smem_fixed_bytes(cap, qcap):
    b = 4 * (3072 + 1) + 4 * 3072 + 4 * (qcap + 1) + 8 * cap + 4 * ((cap + 31) // 32) + 2 * cap + 2 * cap + 4 * cap + \
        2 * (qcap + (qcap & 1)) + 4 * ((qcap + 31) // 32)
    return (b + 15) // 16 * 16


def fit_qcap(cap, nq):
    lo, hi = 1, nq
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        if sbp_smem_fixed_bytes(cap, mid) + 16 * 1024 <= 220 * 1024:
            lo = mid
        else:
            hi = mid - 1
    return lo


def split_chain_scene(depth=60, seed=7):
    """A blocked rule-1 chain straddling the query split of the host guided entry without the histogram: empty padding
    queries (windows in an empty corner of the image) come first, so that the chain's middle falls on the first query of
    the second launch; that launch starts on slots the first one took."""
    qcap = fit_qcap(depth + 1, 10 ** 6)   # the chain's depth + 1 slots are the whole frame
    npad = qcap - depth // 2
    b = Builder(seed)
    for _ in range(npad):
        b.query(W - 50.0, H - 20.0, [])
    chain = add_chain(b, depth, True, 1)
    sc = b.build(Scene("split", 1, facts=dict(chain=chain, qcap=qcap, npad=npad)))
    assert fit_qcap(sc.n, sc.nq) == qcap < sc.nq
    return sc


# ---------------------------------------------------------------------------------------------------------------------
# the scenes realised through the routine-level matchers: a frame of one feature per query at its window centre (F1 /
# Last / KeyFrame) and its map points at (u, v, 1), which the identity pose with fx = fy = 1, cx = cy = 0 projects to
# exactly (u, v) (cv::gemm's float sum of 1 * u, 0 * v, 0 * 1, then + 0)

T_ID = np.hstack([np.eye(3, dtype=np.float32), np.zeros((3, 1), np.float32)])


def f1_keypoints(sc):
    """One level-0 feature per query, at the query's window centre, with the query's angle."""
    k = np.zeros(sc.nq, KP_DTYPE)
    k["x"], k["y"], k["angle"], k["octave"] = sc.qu, sc.qv, sc.qangle, 0
    k["size"], k["response"], k["class_id"] = 31.0, 1.0, -1
    return k


def world_points(sc):
    return np.stack([sc.qu, sc.qv, np.ones(sc.nq, np.float32)], 1).astype(np.float32)


def with_hist(sc, hist):
    h = copy.copy(sc)
    h.hist = hist
    return h


def window_search_view(sc):
    """WindowSearch has no slots occupied on entry: F1 features whose list holds an occupied slot get no map point.
    Returns (f1_has_mp, the scene the sequential loop sees: those queries' lists empty, nothing occupied)."""
    has = np.array([not any(sc.occ[l]) for l in sc.lists], np.uint8)
    v = copy.copy(sc)
    v.lists = [l if h else [] for l, h in zip(sc.lists, has)]
    v.dist = [d if h else [] for d, h in zip(sc.dist, has)]
    v.occ = np.zeros(sc.n, bool)
    return has, v
