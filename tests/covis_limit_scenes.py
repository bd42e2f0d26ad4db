"""Scenes that drive the covisibility graph and its readers to the sizes include/orbfe_bow.h accepts: max_connections 2048,
max_batch 1024 and row caps up to ORBFE_COVIS_OBS_MAX_CAP (8192).  Shared by tests/test_oracle_covis_limits.py (the scenes
reach their sizes; the oracle equals the reference) and tests/test_gpu_covis_limits.py (the device equals the oracle).

Large graphs are stars and bipartite blocks, never cliques: the oracle keeps K x K arrays and re-sorts a whole map on every
AddConnection.  A star's hub shares `weights[i]` points with leaf i; each point is seen by the hub and a group of at most 16
leaves, the groups reshuffled for every point the hub holds of a leaf, so two leaves share few points and the hub's row has
about one cell per leaf.

Every scene carries
  path    the kernel path of orb_slam_b200/csrc/covis.cu it is built for
  keys    its order keys (None: the creation index)
  facts   what the CPU test checks it reaches (counter sizes, events per target, touched slots, list lengths, n0)
and, for refusals, `refused` (the keyframes whose batch must be refused) and `after` (the batch that follows it)."""
import numpy as np

import covis_key_scenes as KM
import covis_scenes as S
import kf_culling_scenes as KS
import local_map_scenes as LS
import observation_scenes as OS

GROUP = 16


def _star_groups(hub, leaves, weights, seed, group=GROUP):
    """one keyframe group per point: the hub and up to `group` leaves; leaf i is in weights[i] of them"""
    rng = np.random.default_rng(seed)
    w = np.asarray(weights, np.int64)
    out = []
    for r in range(int(w.max()) if len(w) else 0):
        have = np.asarray(leaves)[w > r]
        have = have[rng.permutation(len(have))].tolist()
        out += [[hub] + have[j:j + group] for j in range(0, len(have), group)]
    return out


def _cap(nkf, groups, floor=16):
    """the smallest power of two (>= floor) that holds every keyframe's cells"""
    n = np.bincount(np.concatenate([np.asarray(g) for g in groups]), minlength=nkf).max() if groups else 0
    c = floor
    while c < n:
        c *= 2
    return c


class _Free:
    def __init__(self):
        self.f = {}

    def take(self, k):
        v = self.f.get(k, 0)
        self.f[k] = v + 1
        return v


def _points(s, groups, free):
    """one new point per group, seen by every keyframe of the group at its next free feature (reference keyframe: the first)"""
    if not groups:
        return s.npts
    obs = [(j, k, free.take(k)) for j, g in enumerate(groups) for k in g]
    return s.pts([g[0] for g in groups], obs)


def _scene(cls, name, nkf, groups, max_connections, seed, cap=None, **kw):
    s = cls(name, cap or _cap(nkf, groups), seed=seed, max_connections=max_connections, **kw)
    for _ in range(nkf):
        s.kf()
    s.keys, s.facts, s.refused, s.after, s.free = None, {}, None, None, _Free()
    return s


# ---- 1. counter sizes: covis_count_kernel's counter and filtered list sorted by cv_sort at more than one entry per thread

def scene_counter(n, below=False):
    """keyframe 0 the root, 1 the hub, 2 .. n+1 the leaves; the hub's counter holds n entries.  Weights 14 / 15 / 16 with ties
    (or, `below`, 12 / 13 / 14: every weight under 15 and the maximum 14 tied across a third of the keys, so the filtered list
    is the first maximum; interleaved keys make it neither the smallest slot nor the oldest leaf)"""
    hub, leaves = 1, list(range(2, n + 2))
    base = 12 if below else 14
    w = [base + (i * 7) % 3 for i in range(n)]
    groups = _star_groups(hub, leaves, w, seed=n)
    s = _scene(S.Scene, "counter%d%s" % (n, "_below" if below else ""), n + 2, groups, 2048, seed=100 + n)
    _points(s, groups, s.free)
    s.update([hub])
    s.update(leaves[-64:][::-1])   # the hub's map gets its leaves' events (unchanged weights)
    s.update([hub])
    if below:
        s.keys = KM.keys("interleaved", s.nkf)
    s.path = "covis_count_kernel: cv_sort of a counter of %d entries (block 512) and of the filtered list" % n
    s.facts = dict(hub=hub, counter=n, filtered=1 if below else sum(x >= 15 for x in w), weights=w)
    return s


# ---- 2. capacity at every C: refusals of the count kernel (n > C, and the full table at probe == P) and of the plan kernel

def scene_capacity(C, n, weight=15):
    """a hub with n leaves under max_connections C (the hub's update is refused when n > C), and a pair x, y sharing 15
    points with each other alone: x's update is the batch that follows"""
    hub, leaves, x, y = 1, list(range(2, n + 2)), n + 2, n + 3
    groups = _star_groups(hub, leaves, [weight] * n, seed=C + n)
    s = _scene(S.Scene, "capacity_C%d_n%d" % (C, n), n + 4, groups + [[x, y]] * 15, C, seed=200 + n)
    _points(s, groups + [[x, y]] * 15, s.free)
    P = 2 * _pow2ge(C)
    if n > C:
        s.refused = [hub]
    else:
        s.update([hub])
    s.after = [x]
    s.path = "covis_count_kernel: %d distinct covisible keyframes at C = %d (table of P = %d slots%s)" % (
        n, C, P, ", full: probe == P" if n > P else "")
    s.facts = dict(hub=hub, counter=n, C=C, P=P, full=n > P)
    return s


def scene_target_full(C=2048):
    """a target whose map holds C entries receives one more AddConnection from a new keyframe's update: the plan kernel
    refuses the batch"""
    T, leaves, E = 1, list(range(2, C + 2)), C + 2
    groups = _star_groups(T, leaves, [15] * C, seed=C)
    s = _scene(S.Scene, "target_full_C%d" % C, C + 3, groups + [[E, T]] * 15, C, seed=300)
    _points(s, groups, s.free)
    s.update([T])
    _points(s, [[E, T]] * 15, s.free)
    s.refused, s.after = [E], [leaves[3]]
    s.path = "covis_plan_kernel: a target map of %d entries plus one event" % C
    s.facts = dict(target=T, target_map=C, C=C)
    return s


def _pow2ge(n):
    p = 1
    while p < n:
        p <<= 1
    return p


# ---- 3. batches of up to 1024: the apply kernel's event buffer E (Bp) and the plan kernel's touched-slot scan

def scene_batch_hub(nb):
    """nb leaves that each share 15 .. 18 points with a hub: a batch of all nb leaves sends the hub nb events (the hub has
    no call of its own); after more shared points, a batch of nb with the hub's own call in the middle sends it the events
    of the entries after it"""
    hub, leaves = 1, list(range(2, nb + 2))
    w1 = [15 + i % 4 for i in range(nb)]
    g1 = _star_groups(hub, leaves, w1, seed=nb)
    extra = [1 + (i % 3 == 0) for i in range(nb)]   # every leaf's weight changes, a third of them by 2
    g2 = _star_groups(hub, leaves, extra, seed=nb + 1)
    s = _scene(S.Scene, "batch_hub%d" % nb, nb + 2, g1 + g2, 2048, seed=400 + nb)
    _points(s, g1, s.free)
    s.update(leaves)
    _points(s, g2, s.free)
    mid = (nb - 1) // 2
    second = leaves[:mid] + [hub] + leaves[mid:nb - 1]
    s.update(second)
    s.keys = KM.keys("interleaved", s.nkf)
    s.path = "covis_apply_kernel: %d events into one target's E buffer; the own call at batch position %d" % (nb, mid)
    s.facts = dict(hub=hub, batch=nb, events=[nb, nb - 1 - mid], own_at=mid)
    return s


def scene_batch_wide(entries=128, per=12):
    """`entries` keyframes, each with `per` leaves of its own (a bipartite block: 15 points seen by the entry and all its
    leaves), updated in one batch: entries * (1 + per) touched slots"""
    groups, blocks = [], []
    k = 1
    for e in range(entries):
        ent, ls = k, list(range(k + 1, k + 1 + per))
        k += 1 + per
        blocks.append((ent, ls))
        groups += [[ent] + ls] * 15
    s = _scene(S.Scene, "batch_wide%d" % (entries * (1 + per)), k, groups, 2048, seed=500)
    _points(s, groups, s.free)
    order = [b[0] for b in blocks]
    s.update(order[::2] + order[1::2])
    s.update([b[1][0] for b in blocks])   # every first leaf: the entry's map gets an unchanged event
    s.path = "covis_plan_kernel: the touched-slot scan over %d slots (carry across tiles of 1024)" % (entries * (1 + per))
    s.facts = dict(touched=entries * (1 + per), batch=entries)
    return s


# ---- 4. erase: covis_erase_kernel with C blocks and maps of up to 2048 entries

def scene_erase_hub(n=2048):
    """a hub whose map holds n leaves, each leaf's map naming the hub, is erased"""
    hub, leaves = 1, list(range(2, n + 2))
    groups = _star_groups(hub, leaves, [15] * n, seed=7)
    s = _scene(S.Scene, "erase_hub%d" % n, n + 2, groups, 2048, seed=600)
    _points(s, groups, s.free)
    s.update([hub])
    s.erase_kf(hub)
    s.update(leaves[:64])
    s.path = "covis_erase_kernel: %d blocks, one per entry of the erased slot's map" % n
    s.facts = dict(hub=hub, hub_map=n)
    return s


def scene_erase_leaf(n=2048):
    """a hub whose map holds n entries: erase a leaf whose map names the hub (the hub's map re-sorted at n - 1), then a leaf
    the hub names but whose own map does not: its first update, with 20 points shared with keyframe 0 alone, came before
    its 14 points with the hub, and a weight below 15 sends it no event, so the hub's entry goes stale.  (The reference's
    SetBadFlag needs a parent, so every erased keyframe has had its first update.)"""
    hub, leaves = 1, list(range(2, n + 2))
    w = [14 + (i % 3) for i in range(n)]
    named = leaves[1]      # weight 15
    stale = leaves[3]      # weight 14
    groups = _star_groups(hub, leaves, w, seed=8)
    s = _scene(S.Scene, "erase_leaf%d" % n, n + 2, groups + [[stale, 0]] * 20, 2048, seed=700)
    _points(s, [[stale, 0]] * 20, s.free)
    s.update([stale])      # its map: {keyframe 0: 20}
    _points(s, groups, s.free)
    s.update([hub])
    s.update([named])
    s.erase_kf(named)
    s.erase_kf(stale)
    s.update([leaves[5]])  # an event into the map that still names the stale slot
    s.path = "covis_erase_kernel: the hub's map of %d entries re-sorted without the erased leaf; a stale entry" % n
    s.facts = dict(hub=hub, hub_map=n, named=named, stale=stale, weights=w)
    return s


# ---- 6. observations at caps 4096, 4097 and 8192

def scene_obs(cap, n=1100):
    """keyframe 0's row is full: every cell names a point, and the points of its last quarter are the points of its first
    quarter again (the largest index is the observation).  Point 0 is seen by all n keyframes, point 1 by n - 75: their
    lists are longer than 1024 (the sort kernel ranks them in tiles of 1024).  Keyframe 10 is erased at the end."""
    s = OS.ObsScene("obs_cap%d" % cap, cap, seed=800 + cap)
    for _ in range(n):
        s.kf()
    s.keys, s.refused, s.after = KM.keys("random", n), None, None
    q = cap - cap // 4                         # points 2 .. q-1 fill keyframe 0's cells 2 .. q-1, then again from cell q
    obs = [(0, k, 0) for k in range(n)] + [(1, 0, 1)] + [(1, k, 1) for k in range(76, n)]
    for j in range(2, q):
        obs.append((j, 1 + j % (n - 1), 2 + j // (n - 1)))
        obs += [(j, 0, i) for i in range(j, cap, q - 2) if i >= 2]   # ascending cells: the last one written is the largest
    s.pts([0] * q, obs)
    s.update([10])   # its parent, which the reference's SetBadFlag needs
    s.erase_kf(10)
    s.path = "covis_obs_rows_kernel: tables of pow2ge(2 * %d) = %d entries; covis_obs_sort_kernel: lists of %d" % (cap, _pow2ge(2 * cap), n)
    s.facts = dict(cap=cap, full_row=0, long=(0, 1), long_len=(n, n - 75), dup_cells=cap - q)
    return s


# ---- 7. culling: 2048 candidates, rows at cap 8192

def scene_cull(n=2048, window=5, layers=3, fragile=3):
    """K0 (mnId 0, no points), c (the current keyframe) and n candidates.  Every main point is seen by c and a window of
    `window` consecutive candidates (cyclic), `layers` points per window start; every candidate also sees one fragile point,
    seen by c and `fragile` consecutive candidates.  A candidate is redundant while its points keep more than three
    observers: each erase takes an observer from its points, so the list's erases cascade into kept candidates, and the
    second erase among a fragile point's candidates leaves it two observers: bad, partway along the list."""
    k0, c = 0, 1
    cands = list(range(2, n + 2))
    groups = [[c] + [cands[(i + d) % n] for d in range(window)] for i in range(n) for _ in range(layers)]
    groups += [[c] + cands[i:i + fragile] for i in range(0, n, fragile)]
    cap = 8192
    s = _scene(KS.CullScene, "cull%d_cap%d" % (n, cap), n + 2, groups, 2048, seed=900, cap=cap)
    s.free = _Free()
    _points(s, groups, s.free)
    for i in range(0, n, 64):   # every candidate's first update (its parent: c), then c's
        s.update(cands[i:i + 64])
    s.update([c])
    s.cull(c)
    s.keys = KM.keys("interleaved", s.nkf)
    s.path = "covis_cull_check_kernel / covis_cull_kernel: %d candidates, cascades; rows at cap %d" % (n, cap)
    s.facts = dict(current=c, candidates=n, cap=cap)
    return s


# ---- 8. local map: n0 > 1024 counted keyframes, ranked in tiles of 1024

def scene_lm(n, tied_slots=(266, 291, 1025), frame_cells=None):
    """K0 and n keyframes, each seeing a point of its own; a point q seen by the keyframes at `tied_slots`.  The frame names every
    keyframe's point and q twice: n counted keyframes (n0 = n + 1 with K0), the tied ones at 3 votes (the maximum),
    the rest at 1; under interleaved keys the first maximum is neither the first slot nor the oldest.  With frame_cells,
    a second frame of that many cells repeats the first frame's points with NULL cells between."""
    s = _scene(LS.LmScene, "lm%d" % n, n + 1, [], 64, seed=1000 + n, cap=8)
    inv = np.argsort(s.slots())
    tied = [int(inv[t]) for t in tied_slots]   # the keyframes at these slots: the first maximum is in a later tile than the first slot
    s.free = _Free()
    first = _points(s, [[k] for k in range(n + 1)], s.free)
    q = _points(s, [list(tied)], s.free)
    cells = list(range(first, first + n + 1)) + [q, q]
    s.frame(cells)
    if frame_cells:
        big = np.array((cells + [-1]) * (frame_cells // (len(cells) + 1) + 1), np.int32)[:frame_cells]
        s.frame(big)
    s.keys = KM.keys("interleaved", s.nkf)
    s.path = "covis_lm_list_kernel: %d counted slots ranked in tiles of 1024, the maximum tied across tiles" % (n + 1)
    s.facts = dict(n0=n + 1, tied=tied, tied_slots=list(tied_slots), frame_cells=frame_cells)
    return s


COUNTER_SIZES = (511, 512, 513, 1024, 1025, 2047, 2048)


def counter_scenes():
    return [scene_counter(n) for n in COUNTER_SIZES] + [scene_counter(1025, below=True)]


def capacity_scenes():
    out = []
    for C in (1, 1000, 1500, 2048):
        out += [scene_capacity(C, C), scene_capacity(C, C + 1)]
    out += [scene_capacity(6, 17, weight=1), scene_capacity(2048, 4097, weight=1), scene_target_full(2048)]
    return out


def batch_scenes():
    return [scene_batch_hub(1024), scene_batch_hub(1000), scene_batch_wide()]


def erase_scenes():
    return [scene_erase_hub(), scene_erase_leaf()]


def obs_scenes():
    return [scene_obs(4096), scene_obs(4097), scene_obs(8192)]


def lm_scenes():
    return [scene_lm(1025), scene_lm(2048, tied_slots=(968, 1047, 1546, 1947), frame_cells=8192)]
