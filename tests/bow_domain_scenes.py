"""Scenes that put the BoW chain and the Hamming kernels on their decision boundaries (numpy only, no GPU, no reference).

Every distance is made by flipping chosen bits of a base descriptor, so a scene that claims "best 50, second 100" has exactly
those distances.  The builders return plain arrays; tests/test_oracle_bow_domain.py checks that each scene contains the events
it is built for and that the oracle equals the reference's own code on it, tests/test_gpu_bow_domain.py runs the kernels on it.
"""
import numpy as np

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])
F32 = np.float32


# ---- descriptors at exact distances ---------------------------------------------------------------------------------------
def mask(positions):
    """32-byte mask with the given bit positions set (bit p = byte p // 8, bit 7 - p % 8: np.unpackbits order)."""
    bits = np.zeros(256, np.uint8)
    bits[np.asarray(positions, np.int64)] = 1
    return np.packbits(bits)


def away(base, d, rng):
    """`base` with d random bits flipped: at distance exactly d."""
    return base ^ mask(rng.choice(256, d, replace=False))


def hamming(a, b):
    return np.unpackbits(np.bitwise_xor(a, b), axis=-1).sum(axis=-1)


def placements(d):
    """Three placements of d flipped bits: packed from bit 0 (inside one 32-bit word while d <= 32), spread round-robin over
    the eight 32-bit words, and the top bits only."""
    j = np.arange(d)
    return {"packed": j, "spread": (j % 8) * 32 + j // 8, "top": 255 - j}


def distance_set(seed=0):
    """q, t with hamming(q[i], t[i]) == d[i] for d = 0..256 in each of the three placements."""
    rng = np.random.default_rng(seed)
    q, t, dist = [], [], []
    for d in range(257):
        for pos in placements(d).values():
            b = rng.integers(0, 256, 32, dtype=np.uint8)
            q.append(b)
            t.append(b ^ mask(pos))
            dist.append(d)
    return np.array(q, np.uint8), np.array(t, np.uint8), np.array(dist, np.int64)


def knn2_scene(group_size, nq, seed=0):
    """Queries and two groups of `group_size` descriptors.  Group 0 holds planted candidates at distance 10 from query 0 at
    positions (127, 128) and from query 1 at positions 3 and group_size - 1, in two different 128-descriptor chunks (at the
    first and last position when the group is one chunk; at 0 and 1 for 129); every other entry is random.  Returns (q, db, planted)
    with planted = [(query, group, (positions...))]."""
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    db = rng.integers(0, 256, (2 * group_size, 32), dtype=np.uint8)
    planted = []
    g = group_size
    ties = []
    if g >= 129:
        ties.append((0, (127, 128)))
    if g >= 2:
        ties.append((1 % nq, (3, g - 1) if g > 129 else (0, 1) if g == 129 else (0, g - 1)))
    for qi, pos in ties:
        if qi == 0 and nq == 1 and planted:
            break
        for p in pos:
            db[p] = away(q[qi], 10, rng)
        planted.append((qi, 0, pos))
    return q, db, planted


# ---- vocabulary trees from explicit arrays ----------------------------------------------------------------------------------
def tree_arrays(branching):
    """A complete tree with branching[l] children per node at level l, nodes numbered breadth first (the order
    synth.random_vocabulary and Data/ORBvoc.txt use).  Returns (child_ptr, children, level_start, level_size)."""
    size = [1]
    for b in branching:
        size.append(size[-1] * b)
    start = np.concatenate([[0], np.cumsum(size)]).astype(np.int64)
    n = int(start[-1])
    child_ptr = np.full(n + 1, n - 1, np.int64)
    for l, b in enumerate(branching):
        idx = np.arange(start[l], start[l + 1])
        child_ptr[idx] = start[l + 1] + (idx - start[l]) * b - 1
    return child_ptr.astype(np.int32), np.arange(1, n, dtype=np.int32), start, size


def _vocab(branching, node_desc, stopped=()):
    child_ptr, children, start, size = tree_arrays(branching)
    n = len(node_desc)
    L = len(branching)
    word_id = np.full(n, -1, np.int32)
    word_id[start[L]:] = np.arange(size[L], dtype=np.int32)
    weight = np.zeros(n, np.float64)
    weight[start[L]:] = 1.0 + (np.arange(size[L]) % 7) * 0.25
    weight[np.asarray(stopped, np.int64)] = 0.0
    # "k" is only the header of the text format (TemplatedVocabulary::loadFromTextFile reserves k^(L+1) nodes from it)
    return {"node_desc": node_desc, "child_ptr": child_ptr, "children": children, "word_id": word_id, "weight": weight,
            "L": L, "k": 2, "branching": list(branching), "level_start": start}


def parent_of(start, branching, ids):
    ids = np.asarray(ids, np.int64)
    lev = np.searchsorted(start, ids, side="right") - 1
    b = np.array(branching, np.int64)[np.maximum(lev - 1, 0)]
    return np.where(lev == 0, -1, start[np.maximum(lev - 1, 0)] + (ids - start[lev]) // b)


TIE_PAIRS = ((0, 1), (30, 31), (31, 32), (5, 37))


def tie_vocabulary(k, L, seed=0):
    """Root with k children, each child with two children per level down to depth L (a chain when k == 1).  The root's
    children are base ^ M_p with |M_p| = 100, so any two of them differ in an even number of bits; below level 1 both
    children of a node carry their parent's descriptor, so every query ties at list positions (0, 1) on every deeper level."""
    rng = np.random.default_rng(seed)
    branching = [k] + [1 if k == 1 else 2] * (L - 1)
    child_ptr, children, start, size = tree_arrays(branching)
    n = int(start[-1])
    desc = np.zeros((n, 32), np.uint8)
    base = rng.integers(0, 256, 32, dtype=np.uint8)
    for p in range(k):
        desc[1 + p] = base ^ mask(rng.choice(256, 100, replace=False))
    for l in range(2, L + 1):
        ids = np.arange(start[l], start[l + 1])
        desc[ids] = desc[parent_of(start, branching, ids)]
    # the leaf that the "distance 0" query of tie_queries reaches (child k // 2, then child 0 on every level) is a stopped word
    voc = _vocab(branching, desc, stopped=[int(start[L]) + (k // 2) * (size[L] // k)] if k > 1 else ())
    voc["base"] = base
    return voc


def tie_queries(voc, seed=0):
    """Queries for tie_vocabulary: equidistant from the root's children at each pair of TIE_PAIRS that fits and at (0, k-1)
    (half of the differing bits of the two flipped), from all k children at once (the base), at distance 0 from a child and
    at distance 256 from the base's complement ... plus noisy copies of leaves.  Returns (queries, labels)."""
    rng = np.random.default_rng(seed)
    k = voc["branching"][0]
    c = voc["node_desc"][1:1 + k]
    qs, labels = [], []
    pairs = [p for p in TIE_PAIRS if p[1] < k] + ([(0, k - 1)] if k > 1 else [])
    for a, b in pairs:
        diff = np.flatnonzero(np.unpackbits(c[a] ^ c[b]))
        qs.append(c[a] ^ mask(diff[: len(diff) // 2]))
        labels.append("tie %d/%d" % (a, b))
    qs.append(voc["base"].copy()); labels.append("all %d" % k)
    qs.append(c[k // 2].copy()); labels.append("distance 0")
    qs.append(~c[0]); labels.append("complement")
    leaves = voc["node_desc"][voc["level_start"][-2]:]
    for i in rng.integers(0, len(leaves), 6):
        qs.append(away(leaves[i], 6, rng)); labels.append("noisy leaf")
    return np.array(qs, np.uint8), labels


def orbvoc_shape_vocabulary(seed=0):
    """k = 10, L = 6 (1,111,111 nodes): ORBvoc's shape, so leaf and node ids pass 2^16 and 2^20.  Each node is its parent with
    about one bit in eight flipped."""
    rng = np.random.default_rng(seed)
    branching = [10] * 6
    _, _, start, _ = tree_arrays(branching)
    n = int(start[-1])
    desc = np.zeros((n, 32), np.uint8)
    desc[1:11] = rng.integers(0, 256, (10, 32), dtype=np.uint8)
    for l in range(2, 7):
        ids = np.arange(start[l], start[l + 1])
        r = rng.integers(0, 256, (3, len(ids), 32), dtype=np.uint8)
        desc[ids] = desc[parent_of(start, branching, ids)] ^ (r[0] & r[1] & r[2])
    return _vocab(branching, desc, stopped=[int(start[6]) + 5, n - 2])


def orbvoc_queries(voc, n=64, seed=1):
    """Noisy copies of leaves, half of them from the last 62,535 leaves (ids >= 2^20), plus the exact leaf descriptors."""
    rng = np.random.default_rng(seed)
    s6 = int(voc["level_start"][6])
    nn = len(voc["node_desc"])
    ids = np.concatenate([rng.integers(s6, nn, n // 2), rng.integers(1 << 20, nn, n // 2)])
    q = voc["node_desc"][ids].copy()
    q[: n // 2] = [away(x, 4, rng) for x in q[: n // 2]]
    return q, ids


# ---- FeatureVector inputs ---------------------------------------------------------------------------------------------------
FV_CAPS = (1, 2, 31, 1000, 1023, 1024, 1025, 2000, 2047, 2048, 2049, 6144, 6145, 8192, 16383, 16384)


def fv_frames(cap, nnodes, live, seed=0):
    """Leaf / node arrays of one launch (frames x cap) for orbfe_feature_vector_device, vocabulary of `nnodes` nodes whose
    live words are `live` (bool per node).  Frames: counts 0, 1, cap, cap + 5 (clamped), -3 (as 0); then full frames with every
    feature in one node, every feature in its own node, node ids descending with the index, runs of 7 straddling every chunk
    edge, node = index // 1024 (heads exactly at 1024 and 2048), and node ids 0 / 2^31 - 1.  Frames 0-4 mix live, stopped and
    out-of-range leaf ids (-1, nnodes, nnodes + 100)."""
    rng = np.random.default_rng(seed)
    live_ids = np.flatnonzero(live)
    dead_ids = np.flatnonzero(~live)
    counts = [0, 1, cap, cap + 5, -3, cap, cap, cap, cap, cap, cap]
    F = len(counts)
    leaf = live_ids[rng.integers(0, len(live_ids), (F, cap))].astype(np.int32)
    i = np.arange(cap)
    node = np.zeros((F, cap), np.int64)
    node[:5] = rng.integers(0, max(2, cap // 3), (5, cap))
    bad = rng.random((5, cap)) < 0.15
    leaf[:5][bad] = rng.choice(np.concatenate([dead_ids, [-1, nnodes, nnodes + 100]]), int(bad.sum()))
    node[5] = 77
    node[6] = i
    node[7] = cap - i
    node[8] = (i + 3) // 7
    node[9] = i // 1024
    node[10] = np.where(i % 3 == 0, 0, 2 ** 31 - 1)
    node[10, 1::5] = rng.integers(1, 1000, len(node[10, 1::5]))
    return leaf, node.astype(np.int32), np.array(counts, np.int32)


def fv_numpy(leaf, node, count, cap, live):
    """DBoW2's FeatureVector restated: features with a live leaf, grouped by node id, ascending; index order inside a node."""
    n = min(max(int(count), 0), cap)
    lf = leaf[:n].astype(np.int64)
    ok = (lf >= 0) & (lf < len(live))
    ok[ok] = live[lf[ok]]
    kept = np.flatnonzero(ok).astype(np.int32)
    nd = node[:n][kept].astype(np.int64)
    order = np.argsort(nd, kind="stable")
    ids, cnt = np.unique(nd, return_counts=True)
    return ids.astype(np.int32), np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32), kept[order]


# ---- frame stores for SearchByBoW / SearchForTriangulation ----------------------------------------------------------------
class Frame:
    """One frame of a matcher scene: descriptors, keypoints, per-feature flag (SearchByBoW: has a good map point;
    SearchForTriangulation: has a map point) and node id.  Unused slots are random descriptors in a node of their own side."""

    def __init__(self, n, filler_node, seed):
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        self.kps = np.zeros(n, KP_DTYPE)
        self.kps["x"], self.kps["y"] = 320.0, 240.0
        self.flag = np.zeros(n, np.uint8)
        self.node = np.full(n, filler_node, np.int32)
        self.descending = set()
        self.next = 0

    def put(self, desc, node, angle=0.0, flag=0, x=320.0, y=240.0, octave=0, at=None):
        i = self.next if at is None else at
        if at is None:
            self.next += 1
        self.desc[i], self.node[i], self.flag[i] = desc, node, flag
        self.kps[i]["angle"], self.kps[i]["x"], self.kps[i]["y"], self.kps[i]["octave"] = angle, x, y, octave
        return i

    def fv(self):
        order = np.argsort(self.node, kind="stable").astype(np.int32)
        ids, cnt = np.unique(self.node, return_counts=True)
        ptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
        for k, nid in enumerate(ids):
            if int(nid) in self.descending:
                order[ptr[k]:ptr[k + 1]] = order[ptr[k]:ptr[k + 1]][::-1]
        return ids.astype(np.int32), ptr, order


class Expect:
    """What a scene is built for: (i1, i2) = side-1 feature i1 matches side-2 feature i2 (-1: no match) under `when`."""

    def __init__(self):
        self.rows = []

    def add(self, label, i1, i2, **when):
        self.rows.append((label, int(i1), int(i2), when))

    def applicable(self, **run):
        return [(lab, i1, i2) for lab, i1, i2, w in self.rows if all(run.get(k) == v for k, v in w.items())]


def match_of(variant, out, i1):
    """The side-2 match of side-1 feature i1 in an output row (variant 0 rows are indexed by side 2)."""
    if variant == 1:
        return int(out[i1])
    hit = np.flatnonzero(out == i1)
    return int(hit[0]) if len(hit) else -1


BOW_RATIOS = (0.75, 0.6, 1.25)


def bow_boundary_pair(n=2000, seed=0):
    """One (side 1, side 2) pair whose common nodes each hold one SearchByBoW rule at its boundary (orientation off).
    Side-2 flags are the KeyFrame-vs-KeyFrame validity; side-1 flags are all set except for one node."""
    rng = np.random.default_rng(seed)
    f1, f2 = Frame(n, 1 << 30, seed + 1), Frame(n, (1 << 30) + 1, seed + 2)
    f2.flag[:] = 1
    E = Expect()
    node = iter(range(10, 10 ** 6))

    def cands(q, dists, nid, valid=None):
        return [f2.put(away(q, d, rng), nid, flag=1 if valid is None else valid[k]) for k, d in enumerate(dists)]

    def query(nid, flag=1):
        q = rng.integers(0, 256, 32, dtype=np.uint8)
        return q, f1.put(q, nid, flag=flag)

    # TH_LOW (<= 50 for KeyFrame vs Frame, < 50 for KeyFrame vs KeyFrame)
    for d in (49, 50, 51):
        nid = next(node)
        q, i1 = query(nid)
        c = cands(q, [d, 100], nid)
        for v in (0, 1):
            ok = d < 50 or (d == 50 and v == 0)
            E.add("TH_LOW %d v%d" % (d, v), i1, c[0] if ok else -1, variant=v)
    # the ratio test in float: 0.75f*40 == 30 exactly (reject), 0.6f*50 = 30.000002f (accept), ties, a lone candidate
    for (b, s), res in (((30, 40), {0.75: 0, 0.6: -1, 1.25: 0}), ((30, 41), {0.75: 0, 0.6: -1, 1.25: 0}),
                        ((30, 50), {0.75: 0, 0.6: 0, 1.25: 0}), ((30, 30), {0.75: -1, 0.6: -1, 1.25: 0})):
        nid = next(node)
        q, i1 = query(nid)
        c = cands(q, [b, s], nid)
        for r, k in res.items():
            ok = k == 0 and (r == 1.25 or b < F32(r) * F32(s))
            E.add("ratio %d/%d at %g" % (b, s, r), i1, c[0] if ok else -1, nnratio=r)
    nid = next(node)
    q, i1 = query(nid)
    c = cands(q, [30], nid)
    E.add("lone candidate", i1, c[0])
    # a lone valid candidate among invalid ones: KeyFrame vs KeyFrame sees INT_MAX as the second, KeyFrame vs Frame sees 31
    nid = next(node)
    q, i1 = query(nid)
    c = cands(q, [30, 31], nid, valid=[1, 0])
    E.add("lone valid v1", i1, c[0], variant=1)
    E.add("lone valid v0 0.75", i1, -1, variant=0, nnratio=0.75)
    # every other candidate already matched
    nid = next(node)
    q, i1a = query(nid)
    i1b = f1.put(q, nid, flag=1)
    c = cands(q, [10, 31], nid)
    E.add("first of two", i1a, c[0], nnratio=0.75)
    E.add("second takes the lone rest", i1b, c[1], nnratio=0.75)
    # node lengths around the 32 register candidates; best / runner-up in the same lane or in different lanes
    for L, pairs in ((1, [(0, None)]), (31, [(30, 0)]), (32, [(0, 31), (31, 30)]), (33, [(0, 32), (32, 1)]),
                     (63, [(5, 37), (40, 2)]), (64, [(63, 31), (33, 34)]), (65, [(64, 0), (1, 64)]),
                     (300, [(299, 267), (150, 151), (7, 295)])):
        for pb, ps in pairs:
            nid = next(node)
            q, i1 = query(nid)
            d = list(rng.integers(40, 120, L))
            d[pb] = 20
            if ps is not None:
                d[ps] = 22
            c = cands(q, d, nid)
            E.add("length %d best %d second %s at 1.25" % (L, pb, ps), i1, c[pb], nnratio=1.25)
            E.add("length %d best %d second %s at 0.75" % (L, pb, ps), i1, c[pb] if ps is None else -1, nnratio=0.75)
    # equal best distances: the first list position wins (observable when nnratio > 1)
    for a, b in ((0, 1), (31, 32), (5, 37), (40, 41)):
        nid = next(node)
        q, i1 = query(nid)
        d = list(rng.integers(40, 120, 50))
        d[a] = d[b] = 20
        c = cands(q, d, nid)
        E.add("tie %d/%d" % (a, b), i1, c[a], nnratio=1.25)
        E.add("tie %d/%d rejected" % (a, b), i1, -1, nnratio=0.75)
    # contention: side-1 features of one node share their best side-2 feature; list order decides, the later ones fall back
    nid = next(node)
    q, i1a = query(nid)
    i1b, i1c = f1.put(q, nid, flag=1), f1.put(q, nid, flag=1)
    c = cands(q, [60, 10, 70, 14, 30, 90], nid)
    E.add("contention 1", i1a, c[1], nnratio=0.75)
    E.add("contention 2", i1b, c[3], nnratio=0.75)
    E.add("contention 3", i1c, c[4], nnratio=0.75)
    nid = next(node)
    q, i1a = query(nid)
    i1b = f1.put(q, nid, flag=1)
    c = cands(q, [10, 20, 22, 80], nid)
    E.add("contention fallback rejected 1", i1a, c[0], nnratio=0.75)
    E.add("contention fallback rejected 2", i1b, -1, nnratio=0.75)
    # side-2 validity: KeyFrame vs KeyFrame skips the invalid best, KeyFrame vs Frame does not look
    nid = next(node)
    q, i1 = query(nid)
    c = cands(q, [10, 20, 40], nid, valid=[0, 1, 1])
    E.add("invalid best v1", i1, c[1], variant=1, nnratio=0.75)
    E.add("invalid best v0", i1, c[0], variant=0, nnratio=0.75)
    # an invalid side-1 feature is never matched
    nid = next(node)
    q, i1 = query(nid, flag=0)
    cands(q, [5], nid)
    E.add("invalid side 1", i1, -1)
    # a node only side 1 has, and one only side 2 has
    query(next(node))
    f2.put(rng.integers(0, 256, 32, dtype=np.uint8), next(node))
    assert f1.next <= n and f2.next <= n
    return f1, f2, E


# ---- rotation histogram ---------------------------------------------------------------------------------------------------
def rot_bin(a1, a2):
    """The matchers' bin: rot = a1 - a2 (+360 if negative) in float, round(rot * (1.0f/30)) half away from zero, 30 -> 0."""
    rot = F32(F32(a1) - F32(a2))
    if rot < 0:
        rot = F32(rot + F32(360))
    x = F32(rot * F32(F32(1) / F32(30)))
    b = int(np.floor(np.float64(x) + 0.5))
    return 0 if b == 30 else b


def rot_bin_div(a1, a2):
    """The same bin with rot / 30 (a correctly rounded float division) in place of rot * (1.0f/30)."""
    rot = F32(F32(a1) - F32(a2))
    if rot < 0:
        rot = F32(rot + F32(360))
    b = int(np.floor(np.float64(F32(rot / F32(30))) + 0.5))
    return 0 if b == 30 else b


def rotation_sweep():
    """(a1, a2) angle pairs: rot at every 30k + 15 and the three floats on each side, negative differences that wrap to the
    same values, and differences just below 360 (a2 = 0 and a1 one float below 360; a1 = 0 and a tiny a2)."""
    out = []
    for k in range(12):
        b = F32(30 * k + 15)
        vals = [b]
        lo = hi = b
        for _ in range(3):
            lo, hi = np.nextafter(lo, F32(0)), np.nextafter(hi, F32(400))
            vals += [lo, hi]
        for v in vals:
            out.append((F32(v), F32(0)))
        # a negative difference of about b - 360, which the +360 wraps back to about b
        a1 = F32(2.5)
        out.append((a1, F32(a1 + F32(F32(360) - b))))
    out.append((np.nextafter(F32(360), F32(0)), F32(0)))
    out.append((F32(0), F32(1e-6)))
    out.append((F32(0), F32(359.99997)))
    return out


def rotation_pair(matches, seed, kind="bow"):
    """A pair in which match m = one common node with one side-1 feature of angle a1 and one side-2 candidate of angle a2 at
    distance 5 (accepted by every rule): `matches` is a list of (a1, a2).  For kind == "tri" the keypoints lie on the
    epipolar line of F12 = [[0,0,0],[0,0,0],[0,1,0]] (y2 = 0) and no feature has a map point."""
    rng = np.random.default_rng(seed)
    n = max(len(matches), 1)
    f1, f2 = Frame(n, 1 << 30, seed + 1), Frame(n, (1 << 30) + 1, seed + 2)
    pairs = []
    for m, (a1, a2) in enumerate(matches):
        q = rng.integers(0, 256, 32, dtype=np.uint8)
        if kind == "bow":
            i1 = f1.put(q, 100 + m, angle=a1, flag=1)
            i2 = f2.put(away(q, 5, rng), 100 + m, angle=a2, flag=1)
        else:
            i1 = f1.put(q, 100 + m, angle=a1, x=50.0 + m, y=60.0)
            i2 = f2.put(away(q, 5, rng), 100 + m, angle=a2, x=70.0 + m, y=0.0)
        pairs.append((i1, i2))
    return f1, f2, pairs


def cluster(bin_, count):
    return [(F32(30 * bin_), F32(0))] * count


THREE_MAXIMA_SHAPES = {
    "max2 == 0.1 max1": {0: 30, 5: 3},
    "max2 below": {0: 30, 5: 2},
    "max3 == 0.1 max1": {0: 30, 4: 5, 8: 3},
    "max3 below": {0: 30, 4: 5, 8: 2},
    "equal counts": {7: 10, 3: 10, 9: 10, 11: 10},
    "single bin": {4: 7},
}


def three_maxima_keep(counts):
    """ComputeThreeMaxima over bin counts (first maximum wins ties, float 0.1f * max1 cut): the set of kept bins."""
    max1 = max2 = max3 = 0
    i1 = i2 = i3 = -1
    for i in range(30):
        s = counts.get(i, 0)
        if s > max1:
            max3, max2, max1, i3, i2, i1 = max2, max1, s, i2, i1, i
        elif s > max2:
            max3, max2, i3, i2 = max2, s, i2, i
        elif s > max3:
            max3, i3 = s, i
    if F32(max2) < F32(F32(0.1) * F32(max1)):
        i2 = i3 = -1
    elif F32(max3) < F32(F32(0.1) * F32(max1)):
        i3 = -1
    return {i for i in (i1, i2, i3) if i >= 0}


def rotation_jobs():
    """Rotation scenes: (name, matches, kept) with kept[m] = whether match m survives the histogram.  Each swept angle pair
    is run twice, next to a cluster of 11 matches in its own bin and in the neighbouring bin across the boundary (a single
    match beside 11 is dropped, so the swept match survives exactly when it falls in the cluster's bin)."""
    jobs = []
    for name, shape in THREE_MAXIMA_SHAPES.items():
        matches = [m for b, c in sorted(shape.items()) for m in cluster(b, c)]
        keep = three_maxima_keep(shape)
        jobs.append((name, matches, [rot_bin(*m) in keep for m in matches]))
    for a1, a2 in rotation_sweep():
        b = rot_bin(a1, a2)
        rot = F32(F32(a1) - F32(a2))
        rot = F32(rot + F32(360)) if rot < 0 else rot
        other = b - 1 if np.float64(rot) < 30.0 * b else b + 1
        for cb in (b, other):
            matches = cluster(cb % 30, 11) + [(a1, a2)]
            jobs.append(("sweep %r-%r next to bin %d" % (float(a1), float(a2), cb), matches, [True] * 11 + [cb == b]))
    return jobs


# ---- SearchForTriangulation -----------------------------------------------------------------------------------------------
F12_LINE_Y = np.array([0, 0, 0, 0, 0, 0, 0, 1, 0], np.float32)   # row-major [[0,0,0],[0,0,0],[0,1,0]]: line (0,1,0), dsqr = y2^2


def sigma2(nlevels, scale=1.2):
    """KeyFrame::GetSigma2: squared per-level scale factors, accumulated in float as ORBextractor does."""
    sf = [F32(1.0)]
    for _ in range(1, nlevels):
        sf.append(F32(sf[-1] * F32(scale)))
    return np.array([s * s for s in sf], np.float32)


def epipolar_edges(sig2):
    """Per level l: the y2 values around the CheckDistEpipolarLine threshold on F12_LINE_Y: the largest float y2 with
    (double)(y2*y2 in float) < 3.84 * (double)sigma2[l], the next float up, and one float further on each side."""
    out = []
    for l, s in enumerate(sig2):
        thr = 3.84 * float(s)
        y = F32(np.sqrt(thr))
        while float(F32(y * y)) >= thr:
            y = np.nextafter(y, F32(0))
        while float(F32(np.nextafter(y, F32(1e9)) ** 2)) < thr:
            y = np.nextafter(y, F32(1e9))
        up = np.nextafter(y, F32(1e9))
        out += [(l, np.nextafter(y, F32(0)), True), (l, y, True), (l, up, False), (l, np.nextafter(up, F32(1e9)), False)]
    return out


def tri_boundary_pair(n=700, nlevels=8, seed=0):
    """One pair for SearchForTriangulation on F12_LINE_Y (orientation off): TH_LOW 50/51, DistTh = 2 * best at and above,
    best 0, the epipolar threshold at every level, ties by feature index in descending-listed nodes and across the register
    and streaming halves, side-2 candidates with a map point, side-1 features with a map point."""
    rng = np.random.default_rng(seed)
    f1, f2 = Frame(n, 1 << 30, seed + 1), Frame(n, (1 << 30) + 1, seed + 2)
    sig2 = sigma2(nlevels)
    E = Expect()
    node = iter(range(10, 10 ** 6))
    FAR = 100.0   # y2 = 100 fails the epipolar test at every level but the last ones of 32

    def query(nid, mp=0):
        q = rng.integers(0, 256, 32, dtype=np.uint8)
        return q, f1.put(q, nid, flag=mp, x=float(rng.uniform(10, 600)), y=float(rng.uniform(10, 400)))

    def cand(q, d, nid, y=0.0, mp=0, octave=0, at=None):
        return f2.put(away(q, d, rng), nid, flag=mp, x=float(rng.uniform(10, 600)), y=y, octave=octave, at=at)

    for d, ok in ((50, True), (51, False)):
        nid = next(node)
        q, i1 = query(nid)
        c = cand(q, d, nid)
        E.add("TH_LOW %d" % d, i1, c if ok else -1)
    for best, d2, ok in ((20, 40, True), (20, 41, False), (0, 1, False), (0, 0, True), (25, 50, True)):
        nid = next(node)
        q, i1 = query(nid)
        cand(q, best, nid, y=FAR)          # the best fails the epipolar test
        c = cand(q, d2, nid)
        cand(q, 60, nid)
        E.add("DistTh best %d cand %d" % (best, d2), i1, c if ok else -1)
    for l, y2, ok in epipolar_edges(sig2):
        nid = next(node)
        q, i1 = query(nid)
        c = cand(q, 10, nid, y=float(y2), octave=l)
        E.add("epipolar level %d y2 %r" % (l, float(y2)), i1, c if ok else -1)
    # ties by feature index, whatever the list order: descending lists, and a 40-item list (register and streaming halves)
    for L, (pa, pb) in ((2, (0, 1)), (40, (3, 35)), (40, (35, 3)), (70, (64, 2))):
        nid = next(node)
        q, i1 = query(nid)
        ids = [cand(q, int(rng.integers(52, 120)), nid) for _ in range(L)]
        f2.desc[ids[pa]] = away(q, 15, rng)
        f2.desc[ids[pb]] = away(q, 15, rng)
        if L != 70:
            f2.descending.add(nid)
        E.add("tie %d/%d in %d" % (pa, pb, L), i1, min(ids[pa], ids[pb]))
    # map points: a side-2 best with a map point is skipped; a side-1 feature with a map point is not matched
    nid = next(node)
    q, i1 = query(nid)
    cand(q, 5, nid, mp=1)
    c = cand(q, 9, nid)
    E.add("side-2 map point skipped", i1, c)
    nid = next(node)
    q, i1 = query(nid, mp=1)
    cand(q, 5, nid)
    E.add("side-1 map point", i1, -1)
    # contention: the second side-1 feature takes the next free candidate
    nid = next(node)
    q, i1a = query(nid)
    i1b = f1.put(q, nid, x=f1.kps[i1a]["x"], y=f1.kps[i1a]["y"])
    ca, cb = cand(q, 8, nid), cand(q, 12, nid)
    E.add("contention 1", i1a, ca)
    E.add("contention 2", i1b, cb)
    assert f1.next <= n and f2.next <= n
    return f1, f2, E, sig2


def big_pair(kind, cap=65535, seed=0):
    """Side-2 matches at indices >= 32768 and at 65534 in frames of `cap` features (SearchByBoW: variant-0 rows indexed by
    65534; triangulation: the idx2 in the key's low 16 bits).  For triangulation tied candidates at 65532, 50000 and 32769
    must resolve to 32769."""
    rng = np.random.default_rng(seed)
    f1, f2 = Frame(cap, 1 << 30, seed + 1), Frame(cap, (1 << 30) + 1, seed + 2)
    if kind == "bow":
        f1.flag[:] = 1
        f2.flag[:] = 1
    E = Expect()
    at = [32768, 40000, 65534, 65533]
    for m, i2 in enumerate(at):
        q = rng.integers(0, 256, 32, dtype=np.uint8)
        i1 = f1.put(q, 50 + m, flag=1 if kind == "bow" else 0, at=cap - 1 - m if m % 2 else m)
        f2.put(away(q, 7, rng), 50 + m, flag=1 if kind == "bow" else 0, y=0.0, at=i2)
        E.add("index %d" % i2, i1, i2)
    if kind == "tri":
        q = rng.integers(0, 256, 32, dtype=np.uint8)
        i1 = f1.put(q, 99, at=100)
        d = away(q, 9, rng)
        for i2 in (65532, 32769, 50000):
            f2.put(d, 99, y=0.0, at=i2)
        f2.descending.add(99)
        E.add("tie 65532/32769", i1, 32769)
    return f1, f2, E


# ---- ComputeDistinctiveDescriptors ----------------------------------------------------------------------------------------
DISTINCTIVE_SIZES = (1, 2, 3, 4, 31, 32, 33, 64, 65, 257, 1000)


def edge_triangle(m, rng):
    """Three observations [C, A, B] with d(A, B) = m, d(A, C) = m + 1 and d(B, C) > m: rows A and B have the least median m
    (A, position 1, wins), row C a larger one.  Valid for m <= 170."""
    o = max(0, 2 * m - 255)
    assert m + 1 > 2 * o and m - o + m + 1 <= 256
    base = rng.integers(0, 256, 32, dtype=np.uint8)
    perm = rng.permutation(256)
    A = base
    B = base ^ mask(perm[:m])
    C = base ^ mask(perm[m - o: 2 * m + 1 - o])
    return np.stack([C, A, B])


def edge_row0(m, rng):
    """Three observations [X, A, B] with d(X, A) = m, d(X, B) = m + 1 and d(A, B) = 1: row X has median m, rows A and B median 1,
    so A (position 1) wins unless row X's median is computed as 1 or less.  Valid for 2 <= m <= 255."""
    perm = rng.permutation(256)
    A = rng.integers(0, 256, 32, dtype=np.uint8)
    return np.stack([A ^ mask(perm[:m]), A, A ^ mask(perm[m:m + 1])])


def distinctive_groups(seed=0):
    """(label, descriptors) groups: random noisy groups of every size in DISTINCTIVE_SIZES, all identical, complement pairs
    (medians of 256, the last histogram bin), equal least medians away from row 0, least medians on both sides of every
    9-bin lane edge up to 170/171, and a row-0 median on both sides of every lane edge 8/9 ... 251/252 (edge_row0).

    No group has a least median above 170: if every row's median is >= m, greedily picking a row, then a row at >= m from it,
    then a row at >= m from both (each row has at most k - 1 others closer than m, and N >= 2k + 1) gives three descriptors
    pairwise >= m apart, and three 256-bit descriptors have pairwise distances summing to at most 512.  So medians in lanes 19
    to 28 are pinned through a row that must not win: a lane that under-reports one moves the argmin off row 1."""
    rng = np.random.default_rng(seed)
    out = []
    for N in DISTINCTIVE_SIZES:
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        flip = (rng.random((N, 256)) < rng.uniform(0.05, 0.3)).astype(np.uint8)
        out.append(("random %d" % N, np.unpackbits(base)[None, :] ^ flip))
        out[-1] = (out[-1][0], np.packbits(out[-1][1], axis=1))
    for N in (1, 5, 40):
        out.append(("identical %d" % N, np.repeat(rng.integers(0, 256, (1, 32), dtype=np.uint8), N, axis=0)))
    b = rng.integers(0, 256, 32, dtype=np.uint8)
    out.append(("complement 2", np.stack([b, ~b])))
    out.append(("complement 3", np.stack([b, ~b, ~b])))
    out.append(("complement 7", np.stack([b, ~b, ~b, b, ~b, ~b, ~b])))
    x = rng.integers(0, 256, 32, dtype=np.uint8)
    out.append(("equal least medians", np.stack([~x, x, x, away(x, 3, rng), ~x])))
    for L in range(19):
        for m in (9 * L + 8, 9 * L + 9):
            if m <= 170:
                out.append(("lane edge %d" % m, edge_triangle(m, rng)))
    for L in range(29):
        for m in (9 * L + 8, 9 * L + 9):
            if m <= 252:
                out.append(("row-0 lane edge %d" % m, edge_row0(m, rng)))
    return out


def medians(g):
    """Per row: the (int)(0.5 * (N - 1))-th smallest distance to the group (self included), as MapPoint.cc:225-240."""
    D = hamming(g[:, None, :], g[None, :, :])
    k = (len(g) - 1) // 2
    return np.sort(D, axis=1)[:, k]
