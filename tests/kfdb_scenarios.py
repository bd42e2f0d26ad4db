"""Scripted operation sequences for the keyframe database (include/orbfe_bow.h orbfe_kfdb_*, oracle/kfdb.py).  An operation is
  ("add", slot, ids, vals) | ("erase", slot) | ("clear",) | ("covis", {slot: [slots]}) |
  ("loop", q_ids, q_vals, connected_slots, min_score) | ("reloc", q_ids, q_vals)
Every sequence keeps covisibility lists free of erased slots (as KeyFrame::SetBadFlag leaves its neighbours), so that the
reference's own KeyFrameDatabase, which holds keyframes rather than slots, can replay it."""
import numpy as np


def _bow(rng, ids):
    ids = np.unique(np.asarray(ids, np.int64)).astype(np.int32)
    v = rng.uniform(0.2, 3.0, len(ids))
    return ids, v / v.sum()


def stale_reloc_sequence():
    """Two relocalisation queries where the second reads a score the first one left: keyframe B is scored by query 1 and only
    touched (one shared word, under the word threshold) by query 2, and B is keyframe A's best covisible.  With the persistent
    mRelocScore the candidate is B; with a score of 0 it is A."""
    rng = np.random.default_rng(7)
    A = _bow(rng, range(0, 100))
    B = _bow(rng, range(100, 200))
    C = _bow(rng, range(300, 400))
    ops = [("add", 0, *A), ("add", 1, *B), ("add", 2, *C), ("covis", {0: [1], 1: [0], 2: []}),
           ("reloc", *B),
           ("reloc", *_bow(rng, list(range(0, 100)) + [100]))]
    return ops


def trajectory(nkf, nwords, words_per_kf, seed, shift=None):
    """BowVectors of keyframes along a trajectory: keyframe k sees a window of a random word sequence (neighbours share most
    words), a quarter of them replaced by random words."""
    rng = np.random.default_rng(seed)
    shift = shift or max(1, words_per_kf // 8)
    track = rng.integers(0, nwords, nkf * shift + words_per_kf * 2)

    def at(pos, s):
        r = np.random.default_rng(s)
        w = track[pos:pos + words_per_kf].copy()
        flip = r.random(len(w)) < 0.25
        w[flip] = r.integers(0, nwords, int(flip.sum()))
        return _bow(r, w)

    return [at(shift * k, seed * 100003 + k) for k in range(nkf)], at


def mixed_sequence(seed, nkf=60, nwords=3000, words_per_kf=120, nops=120):
    """add / erase / covisibility refresh / loop and relocalisation queries interleaved, a clear in the middle and slot reuse."""
    rng = np.random.default_rng(seed)
    bows, at = trajectory(nkf * 3, nwords, words_per_kf, seed)
    K = nkf
    occupied = {}
    ops = []
    nxt = 0

    def refresh(slots):
        lists = {}
        for s in slots:
            if s not in occupied:
                continue
            nb = sorted(occupied, key=lambda o: abs(occupied[o] - occupied[s]))
            nb = [o for o in nb if o != s][:int(rng.integers(0, 11))]
            lists[s] = nb
        if lists:
            ops.append(("covis", lists))

    current_lists = {}
    for step in range(nops):
        r = rng.random()
        free = [s for s in range(K) if s not in occupied]
        if (r < 0.35 or len(occupied) < 8) and free and nxt < len(bows):
            s = int(rng.choice(free))
            ops.append(("add", s, *bows[nxt]))
            occupied[s] = nxt
            nxt += 1
            refresh([s] + list(occupied)[:3])
        elif r < 0.45 and occupied:
            s = int(rng.choice(list(occupied)))
            del occupied[s]
            current_lists.pop(s, None)
            ops.append(("erase", s))
            # its neighbours forget it (KeyFrame::SetBadFlag erases the connections)
            lists = {o: [x for x in current_lists.get(o, []) if x != s] for o in occupied}
            if lists:
                ops.append(("covis", lists))
        elif r < 0.5 and occupied:
            refresh(list(occupied))
        elif r < 0.75 and occupied:
            # a new keyframe revisits an earlier place: noisy copy of an added keyframe's view
            src = int(rng.integers(0, max(nxt, 1)))
            q = at(src * max(1, words_per_kf // 8) + int(rng.integers(0, 5)), 7777 + step)
            conn = [s for s in occupied if rng.random() < 0.15]
            ops.append(("loop", *q, conn, float(rng.choice([0.0, 0.01, 0.05]))))
        elif occupied:
            src = int(rng.integers(0, max(nxt, 1)))
            ops.append(("reloc", *at(src * max(1, words_per_kf // 8) + int(rng.integers(0, 5)), 8888 + step)))
        if step == nops // 2:
            ops.append(("clear",))
            occupied.clear()
            current_lists.clear()
        # keep the lists the last covis op set, for the erase bookkeeping
        if ops and ops[-1][0] == "covis":
            for s, lst in ops[-1][1].items():
                current_lists[s] = [x for x in lst if x in occupied]
    return ops, K


def replay(db, ops, on_query=None):
    """Apply ops to anything with add / erase / clear / set_covisibles / detect (the library wrapper or the oracle); returns the
    outputs of every query as (candidates, words, scores)."""
    out = []
    for op in ops:
        kind = op[0]
        if kind == "add":
            db.add(op[1], op[2], op[3])
        elif kind == "erase":
            db.erase(op[1])
        elif kind == "clear":
            db.clear()
        elif kind == "covis":
            db.set_covisibles(op[1])
        elif kind == "loop":
            out.append(db.detect(0, op[1], op[2], op[3], op[4]))
        else:
            out.append(db.detect(1, op[1], op[2]))
    return out
