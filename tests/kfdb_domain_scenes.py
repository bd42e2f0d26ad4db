"""Keyframe-database scenes on the decision boundaries of KeyFrameDatabase (reference src/KeyFrameDatabase.cc:75-308) and at
the size limits of the resident database (include/orbfe_bow.h orbfe_kfdb_*).  numpy only: op sequences in the format of
kfdb_scenarios.replay, each with the facts it is built to produce and the plausible wrong variants whose outcome it changes.

Values are dyadic, so every L1 score and every float sum is exact or rounds where the scene intends.  Every query word has
the value QV = 2 and no keyframe value exceeds it, so a keyframe's L1 score is the sum of its values on the shared words
(|v - w| - |v| - |w| = -2 min(v, w) for positive values): `kf(words, score)` puts the whole score on the first word and 0
on the rest.  Groups of one scene use disjoint word blocks, so each query touches only its own group.

Facts, per query q:  ("cands", q, slots) the candidate list;  ("words", q, slot, n) and ("score", q, slot, x) the query fields
of a slot (x compared as float32 bits; -1 = not touched);  ("min_common", q, m) minCommonWords, from the words of the touched
keyframes that are not connected to the query.

Variants (tests/test_oracle_kfdb_domain.py runs each on the oracle):  words_ge (words >= minCommon), minscore_gt (si > minScore),
retain_ge (accScore >= 0.75 bestAccScore), best_ge (covisible score >= bestScore), order_slot / order_add / order_word (the
sharing list by slot, by add order alone, by first shared word alone with ties by slot), no_narrow (the score kept in double),
narrow_rz (narrowed toward zero), acc_double (covisibility sum in double), acc_reversed (covisibility list summed last to
first), stale_zero (a relocalisation covisible that was not scored by this query counts 0)."""
import numpy as np

F32 = np.float32
QV = 2.0
NWORDS = 65536          # every scene's word ids are below this (the 16-bit scene needs 65535 words)
VARIANTS = ("words_ge", "minscore_gt", "retain_ge", "best_ge", "order_slot", "order_add", "order_word", "no_narrow", "narrow_rz",
            "acc_double", "acc_reversed", "stale_zero")


def below(x):
    """The float32 below x."""
    return float(np.nextafter(F32(x), F32(-np.inf)))


def above(x):
    return float(np.nextafter(F32(x), F32(np.inf)))


def kf(words, score, extra=()):
    """A BowVector that shares `words` with a query of value QV on every word: L1 score `score` (on the first word), plus
    `extra` words (value 1) no query of the group holds."""
    extra = set(int(w) for w in extra)
    ids = np.array(sorted(set(int(w) for w in words) | extra), np.int32)
    vals = np.array([1.0 if w in extra else 0.0 for w in ids.tolist()])
    vals[int(np.searchsorted(ids, min(words)))] = score
    return ids, vals


class Scene:
    def __init__(self, name, K):
        self.name, self.K = name, K
        self.ops, self.facts, self.kills = [], [], set()
        self.nq = 0
        self.pending = None                          # op index of a query a host call follows (host_* scenes)
        self.compactions = 0                         # of the library's store with max_postings = P (finish())
        self._w = 0
        self._live, self._peak = {}, 0

    def block(self, n):
        """n fresh word ids."""
        self._w += n
        assert self._w <= NWORDS
        return list(range(self._w - n, self._w))

    def add(self, slot, ids, vals):
        ids, vals = np.asarray(ids, np.int32), np.asarray(vals, np.float64)
        assert np.all(np.diff(ids) > 0) and slot not in self._live and 0 <= slot < self.K
        self.ops.append(("add", int(slot), ids, vals))
        self._live[slot] = len(ids)
        self._peak = max(self._peak, sum(self._live.values()))

    def erase(self, slot):
        self.ops.append(("erase", int(slot)))
        self._live.pop(slot, None)

    def clear(self):
        self.ops.append(("clear",))
        self._live.clear()

    def covis(self, lists):
        self.ops.append(("covis", {int(k): [int(x) for x in v] for k, v in lists.items()}))

    def loop(self, ids, vals=None, conn=(), min_score=0.0):
        ids = np.asarray(ids, np.int32)
        self.ops.append(("loop", ids, np.full(len(ids), QV) if vals is None else np.asarray(vals, np.float64), [int(c) for c in conn],
                         float(min_score)))
        self.nq += 1
        return self.nq - 1

    def reloc(self, ids, vals=None):
        ids = np.asarray(ids, np.int32)
        self.ops.append(("reloc", ids, np.full(len(ids), QV) if vals is None else np.asarray(vals, np.float64)))
        self.nq += 1
        return self.nq - 1

    def fact(self, q, kind, *args):
        self.facts.append((kind, q) + args)

    def cands(self, q, slots):
        self.fact(q, "cands", [int(s) for s in slots])

    @property
    def P(self):
        """max_postings for the library: the peak number of live postings, so that an add after an erase that left a hole
        compacts the store (counted in self.compactions, restating the library's allocation)."""
        return max(self._peak, 1)

    def finish(self):
        """Count the store compactions the library makes with max_postings = P (orbfe_kfdb_add: the rows go to the tail, and
        the live rows are compacted first when the tail is full)."""
        P, top, live, begin, ln = self.P, 0, 0, {}, {}
        for op in self.ops:
            if op[0] == "add":
                nw = len(op[2])
                if top + nw > P:
                    self.compactions += 1
                    top = live
                begin[op[1]], ln[op[1]] = top, nw
                top += nw
                live += nw
            elif op[0] == "erase" and op[1] in ln:
                nw = ln.pop(op[1])
                if begin.pop(op[1]) + nw == top:
                    top -= nw
                live -= nw
            elif op[0] == "clear":
                top = live = 0
                begin.clear()
                ln.clear()
        return self


# ---- a. the word threshold: minCommonWords = (int)(maxCommonWords * 0.8f), words > minCommonWords ---------------------------
def word_threshold():
    s = Scene("word_threshold", K=40)
    slot = iter(range(s.K))
    for M in (2, 4, 5, 9, 10, 11, 100, 1000):
        m = int(F32(M) * F32(0.8))
        W = s.block(M)
        X, A, B = next(slot), next(slot), next(slot)
        s.add(X, *kf(W, 1.0))                       # maxCommonWords
        s.add(A, *kf(W[M - m:], 1.0))                # exactly minCommonWords: out
        s.add(B, *kf(W[M - m - 1:], 1.0))            # one more: in
        for q in (s.loop(W), s.reloc(W)):
            s.fact(q, "min_common", m)
            s.fact(q, "words", A, m)
            s.fact(q, "words", B, m + 1)
            s.fact(q, "score", A, 0.0)               # never scored: a fresh keyframe's 0
            s.cands(q, [X, B])
    # maxCommonWords = 1: minCommonWords = 0, every touched keyframe qualifies
    W = s.block(1)
    E = s.block(3)
    P, Q = next(slot), next(slot)
    s.add(P, *kf(W, 0.5, extra=E))
    s.add(Q, *kf(W, 0.5))
    for q in (s.loop(W), s.reloc(W)):
        s.fact(q, "min_common", 0)
        s.cands(q, [P, Q])
    # loop mode: a connected keyframe that shares every word does not raise maxCommonWords and reports 1 word
    W = s.block(10)
    C, X, A, B = next(slot), next(slot), next(slot), next(slot)
    s.add(C, *kf(W, 1.0))
    s.add(X, *kf(W[:5], 1.0))
    s.add(A, *kf(W[1:5], 1.0))                       # 4 = (int)(5 * 0.8f): out
    s.add(B, *kf(W[5:], 1.0))
    q = s.loop(W, conn=[C])
    s.fact(q, "min_common", 4)
    s.fact(q, "words", C, 1)
    s.fact(q, "words", A, 4)
    s.cands(q, [X, B])
    q = s.reloc(W)                                   # the same keyframe unconnected: it sets the threshold
    s.fact(q, "min_common", 8)
    s.fact(q, "words", C, 10)
    s.cands(q, [C])
    s.kills |= {"words_ge"}
    return s.finish()


# ---- b. the minimum score: si >= minScore ------------------------------------------------------------------------------------
def min_score():
    s = Scene("min_score", K=8)
    W = s.block(3)
    P, Q = 0, 1
    s.add(P, *kf(W, 0.25))
    s.add(Q, *kf(W, below(0.25)))
    q = s.loop(W, min_score=0.25)
    s.fact(q, "score", P, 0.25)
    s.fact(q, "score", Q, below(0.25))
    s.cands(q, [P])                                  # si == minScore kept, the float below dropped
    W = s.block(4)
    Z, O, H = 2, 3, 4
    s.add(Z, *kf(W, 0.0))
    s.add(O, *kf(W, 0.5))
    s.add(H, *kf(W, 1.0))
    for m, want in ((-np.inf, [H]), (-0.0, [H]), (np.inf, []), (np.nan, [])):
        q = s.loop(W, min_score=m)
        s.fact(q, "score", Z, -0.0)                  # every qualifying keyframe is scored, kept or not; -(0.0) / 2 = -0
        s.fact(q, "score", H, 1.0)
        s.cands(q, want)
    # a keyframe of score -0 alone, at minScore -0.0: kept by si >= minScore, but -0 > 0.75 * -0.0 fails
    W = s.block(2)
    s.add(5, *kf(W, 0.0))
    q = s.loop(W, min_score=-0.0)
    s.cands(q, [])
    s.kills |= {"minscore_gt"}
    return s.finish()


# ---- c. narrowing of the double L1 score to float ----------------------------------------------------------------------------
def narrowing():
    s = Scene("narrowing", K=8)
    lo, hi = 0.5 + 2.0 ** -25, 0.5 + 3 * 2.0 ** -25  # halfway between floats: to 0.5 (even) and up to 0.5 + 2^-23 (even)
    W = s.block(3)
    A, B = 0, 1
    s.add(A, *kf(W, lo))
    s.add(B, *kf(W, hi))
    q = s.loop(W, min_score=0.5 + 2.0 ** -23)
    s.fact(q, "score", A, 0.5)
    s.fact(q, "score", B, 0.5 + 2.0 ** -23)
    s.cands(q, [B])                                  # narrowed B equals minScore; its double, or B toward zero, is below
    # retain: B' is the best; 0.75f * (0.5 + 2^-23) = 0.375 + 3 * 2^-25 is C's score exactly, so C is dropped
    W = s.block(3)
    B2, C = 2, 3
    s.add(B2, *kf(W, hi))
    s.add(C, *kf(W, 0.375 + 3 * 2.0 ** -25))
    q = s.reloc(W)
    s.fact(q, "score", B2, 0.5 + 2.0 ** -23)
    s.cands(q, [B2])
    s.kills |= {"no_narrow", "narrow_rz", "retain_ge"}
    return s.finish()


# ---- d. the retain threshold and the float covisibility sum -------------------------------------------------------------------
def retain():
    s = Scene("retain", K=16)
    # accScore == 0.75f * bestAccScore is dropped, one float above is kept
    W = s.block(3)
    P, Q, R = 0, 1, 2
    s.add(P, *kf(W, 1.0))
    s.add(Q, *kf(W, 0.75))
    s.add(R, *kf(W, above(0.75)))
    q = s.reloc(W)
    s.cands(q, [P, R])
    # in list order 2^-24 + 2^-24 + 1 = 1 + 2^-23; summed last to first it is 1.  0.75f * (1 + 2^-23) = 0.75 + 2^-23 drops Y
    W = s.block(3)
    P2, C1, C2, Y = 3, 4, 5, 6
    s.add(P2, *kf(W, 2.0 ** -24))
    s.add(C1, *kf(W, 2.0 ** -24))
    s.add(C2, *kf(W, 1.0))
    s.add(Y, *kf(W, above(0.75)))
    s.covis({P2: [C1, C2]})
    q = s.reloc(W)
    s.cands(q, [C2])
    # in float 1 + 2^-24 + 2^-24 = 1; in double 1 + 2^-23, which would drop Y'
    W = s.block(3)
    P3, D1, D2, Y3 = 7, 8, 9, 10
    s.add(P3, *kf(W, 1.0))
    s.add(D1, *kf(W, 2.0 ** -24))
    s.add(D2, *kf(W, 2.0 ** -24))
    s.add(Y3, *kf(W, above(0.75)))
    s.covis({P3: [D1, D2]})
    q = s.loop(W)
    s.cands(q, [P3, Y3])
    s.kills |= {"retain_ge", "acc_reversed", "acc_double", "no_narrow"}
    return s.finish()


# ---- e. the best covisible and the first entry naming a keyframe --------------------------------------------------------------
def best_covisible():
    s = Scene("best_covisible", K=1610)
    # a covisible whose score equals si: the keyframe itself stays best
    W = s.block(3)
    s.add(0, *kf(W, 0.5))
    s.add(1, *kf(W, 0.5))
    s.covis({0: [1]})
    s.cands(s.reloc(W), [0])
    # two covisibles of equal score: the first in the list wins
    W = s.block(3)
    s.add(2, *kf(W, 0.25))
    s.add(3, *kf(W, 0.5))
    s.add(4, *kf(W, 0.5))
    s.covis({2: [3, 4]})
    s.cands(s.reloc(W), [3])
    # 1600 entries: entries 3 and 1500 (list positions) both name keyframe B, entry 1000 names D; only entry 3 emits B
    W = s.block(2)
    base, n = 5, 1600
    slot_at = [base + (7 * i + 11) % n for i in range(n)]
    B, D = slot_at[1200], slot_at[1300]
    for i in range(n):
        s.add(slot_at[i], *kf(W, 1.0 if i in (1200, 1300) else 0.5))
    s.covis({slot_at[3]: [B], slot_at[1500]: [B], slot_at[1000]: [D]})
    for q in (s.reloc(W), s.loop(W)):
        s.cands(q, [B, D])
    s.kills |= {"best_ge"}
    return s.finish()


# ---- f. relocalisation only: stale and fresh mRelocScore, zero values ---------------------------------------------------------
def reloc_state():
    s = Scene("reloc_state", K=16)
    WA, WB = s.block(5), s.block(5)
    A, B = 0, 1
    s.add(A, *kf(WA, 0.5))
    s.add(B, *kf(WB, 1.0))
    s.covis({A: [B]})
    q = s.reloc(WB)                                   # scores B: mRelocScore 1
    s.fact(q, "score", B, 1.0)
    vals = np.full(len(WB), QV)
    vals[0] = 0.25
    q = s.loop(WB, vals)                              # scores B in loop mode: mLoopScore 0.25, not read below
    s.fact(q, "score", B, 0.25)
    q = s.reloc(WA + [WB[0]])                         # B touched, one word: its stale mRelocScore 1 makes it A's best
    s.fact(q, "words", B, 1)
    s.fact(q, "score", B, 1.0)
    s.cands(q, [B])
    s.erase(B)                                        # B erased and a new keyframe in its slot: a fresh 0
    s.add(B, *kf(WB, 1.0))
    s.covis({A: [B]})
    q = s.reloc(WA + [WB[0]])
    s.fact(q, "words", B, 1)
    s.fact(q, "score", B, 0.0)
    s.cands(q, [A])
    # every value zero: every keyframe qualifies with score -0 (L1Scoring returns -0.0 / 2) and none is a candidate
    W = s.block(4)
    for k in range(2, 6):
        ids, vals = kf(W, 0.0)
        s.add(k, ids, vals)
    q = s.reloc(W, np.zeros(len(W)))
    for k in range(2, 6):
        s.fact(q, "words", k, 4)
        s.fact(q, "score", k, -0.0)
    s.cands(q, [])
    s.kills |= {"stale_zero"}
    return s.finish()


# ---- g. loop only: which covisibles add their mLoopScore ----------------------------------------------------------------------
def loop_covisibles():
    s = Scene("loop_covisibles", K=16)
    # a qualified covisible below minScore still adds its mLoopScore: P's 0.5 + 0.25 beats R's 0.55 and drops it
    W = s.block(4)
    P, Q, R = 0, 1, 2
    s.add(P, *kf(W, 0.5))
    s.add(Q, *kf(W, 0.25))
    s.add(R, *kf(W, 0.5 + 2.0 ** -4 - 2.0 ** -6))   # 0.546875
    s.covis({P: [Q]})
    q = s.loop(W, min_score=0.3)
    s.fact(q, "score", Q, 0.25)
    s.cands(q, [P])
    # a covisible touched under the word threshold adds nothing (its mLoopScore 1 is an earlier query's)
    WP, WU = s.block(5), s.block(5)
    P2, U = 3, 4
    s.add(P2, *kf(WP, 0.5))
    s.add(U, *kf(WU, 1.0))
    s.covis({P2: [U]})
    q = s.loop(WU)
    s.fact(q, "score", U, 1.0)
    q = s.loop(WP + [WU[0]])
    s.fact(q, "words", U, 1)
    s.cands(q, [P2])
    # a connected covisible adds nothing
    WP, WC = s.block(5), s.block(5)
    P3, Cn = 5, 6
    s.add(P3, *kf(WP, 0.5))
    s.add(Cn, *kf(WC, 1.0))
    s.covis({P3: [Cn]})
    s.loop(WC)
    q = s.loop(sorted(WP + WC), conn=[Cn])
    s.fact(q, "words", Cn, 1)
    s.fact(q, "score", Cn, 1.0)
    s.cands(q, [P3])
    return s.finish()


# ---- h. the order of lKFsSharingWords: first shared query word, then position in that word's list (add order) -------------------
def list_order():
    s = Scene("list_order", K=8)
    W = s.block(4)
    first1, first0 = [W[1], W[2], W[3]], [W[0], W[2], W[3]]
    a, b, c, d = 2, 0, 3, 1                           # added in this order; a, b share from word 1 on, c, d from word 0
    bows = {a: kf(first1, 0.5), b: kf(first1, 0.5), c: kf(first0, 0.5), d: kf(first0, 0.5)}
    for k in (a, b, c, d):
        s.add(k, *bows[k])
    for q in (s.reloc(W), s.loop(W)):
        s.cands(q, [c, d, a, b])                      # slot order, add order and first-word order all disagree
    s.erase(c)                                        # c again into its slot, a into another: both to the tail
    s.add(c, *bows[c])
    s.erase(a)
    s.add(4, *bows[a])
    for q in (s.reloc(W), s.loop(W)):
        s.cands(q, [d, c, b, 4])
    s.erase(b)                                        # a keyframe of another place in b's slot: the store compacts
    s.add(b, *kf(s.block(3), 0.5))
    for q in (s.reloc(W), s.loop(W)):
        s.cands(q, [d, c, 4])
    s.clear()                                         # a clear, then adds in a new order
    for k, bw in ((5, bows[d]), (6, bows[b]), (0, bows[c]), (7, bows[a])):
        s.add(k, *bw)
    for q in (s.reloc(W), s.loop(W)):
        s.cands(q, [5, 0, 6, 7])
    s.kills |= {"order_slot", "order_add", "order_word"}
    return s.finish()


# ---- i. sizes: qualifying keyframes across the 1024-entry chunks of the order and select kernels -------------------------------
def sizes(n):
    K = n + 5                                         # never a power of two here
    s = Scene("size_%d" % n, K=K)
    W = s.block(2)
    slot_at = [(7919 * i + 13) % K for i in range(n)]
    assert len(set(slot_at)) == n
    keep = [i for i in range(n) if i % 3 != 1]
    for i in range(n):
        s.add(slot_at[i], *kf(W, 1.0 if i % 3 != 1 else 0.5))
    for q in (s.reloc(W), s.loop(W)):
        s.fact(q, "min_common", 1)
        s.cands(q, [slot_at[i] for i in keep])
    s.kills |= {"order_slot"}
    return s.finish()


def tiny(K):
    s = Scene("tiny_K%d" % K, K=K)
    W = s.block(3)
    s.add(K - 1, *kf(W, 0.5))
    s.cands(s.reloc(W), [K - 1])
    q = s.loop(W, conn=[K - 1])
    s.fact(q, "words", K - 1, 1)
    s.cands(q, [])
    if K >= 3:
        s.add(0, *kf(W, 1.0))
        s.add(1, *kf(W[1:], 0.25))
        s.covis({K - 1: [0], 1: [K - 1]})
        s.cands(s.reloc(W), [0])
        s.cands(s.loop(W, conn=[0]), [K - 1])
    s.erase(K - 1)
    s.cands(s.reloc(W), [0] if K >= 3 else [])
    return s.finish()


# ---- j. the 16-bit fields of the packed query state: nq = 65535 -------------------------------------------------------------------
def nq_65535():
    s = Scene("nq_65535", K=3)
    W = s.block(65535)
    F, L, S = 2, 0, 1
    s.add(F, *kf(W, 1.0))                             # every word: 65535 shared words
    s.add(L, *kf(W[-1:], 0.5))                        # only the last: first shared rank 65534
    s.add(S, *kf(W[:1], 0.5))                         # only the first
    q = s.reloc(W)
    s.fact(q, "words", F, 65535)
    s.fact(q, "words", L, 1)
    s.fact(q, "min_common", 52428)
    s.cands(q, [F])
    q = s.loop(W, conn=[F])                           # F connected: minCommonWords 0, S (rank 0) before L (rank 65534)
    s.fact(q, "words", F, 1)
    s.fact(q, "min_common", 0)
    s.cands(q, [S, L])
    s.kills |= {"order_add", "order_slot"}
    return s.finish()


# ---- stream ordering: each query's result depends on the stale score the previous query left -------------------------------------
def stream_chain(n=8):
    """Query k qualifies X_k (score 1 - k/16) and touches X_{k-1} with one word: X_{k-1}'s mRelocScore from query k-1 is
    larger than X_k's, so X_{k-1} is X_k's best covisible and the candidate; run before query k-1 it would count 0."""
    s = Scene("stream_chain", K=n + 1)
    Ws = [s.block(5) for _ in range(n)]
    for k in range(n):
        s.add(k, *kf(Ws[k], 1.0 - k / 16.0))
    s.covis({k: [k - 1] for k in range(1, n)})
    for k in range(n):
        q = s.reloc(Ws[k] if k == 0 else sorted(Ws[k] + [Ws[k - 1][0]]))
        s.cands(q, [max(k - 1, 0)])
    s.kills |= {"stale_zero"}
    return s.finish()


def host_call(kind):
    """A query, then a host call (erase / add / set_covisibles / clear) that would change the query's result had it run
    first, then the same query again.  self.pending is the op index of the first query."""
    s = Scene("host_" + kind, K=8)
    W = s.block(4)
    E, G, H = 0, 1, 2
    s.add(E, *kf(W, 1.0))
    s.add(G, *kf(W, 0.5))
    s.add(H, *kf(W, 0.5))
    s.cands(s.reloc(W), [E])
    s.pending = len(s.ops) - 1
    if kind == "erase":
        s.erase(E)
        after = [G, H]
    elif kind == "add":
        s.add(3, *kf(W, 2.0))
        after = [3]
    elif kind == "covis":
        s.covis({G: [H]})                             # G's sum 1.0 equals E's: both kept
        after = [E, G]
    else:
        s.clear()
        after = []
    s.cands(s.reloc(W), after)
    return s.finish()


def all_scenes():
    return ([word_threshold(), min_score(), narrowing(), retain(), best_covisible(), reloc_state(), loop_covisibles(), list_order()]
            + [sizes(n) for n in (1023, 1024, 1025, 2049, 5000)] + [tiny(1), tiny(3), nq_65535(), stream_chain()]
            + [host_call(k) for k in ("erase", "add", "covis", "clear")])


SCENE_NAMES = ["word_threshold", "min_score", "narrowing", "retain", "best_covisible", "reloc_state", "loop_covisibles", "list_order",
               "size_1023", "size_1024", "size_1025", "size_2049", "size_5000", "tiny_K1", "tiny_K3", "nq_65535", "stream_chain",
               "host_erase", "host_add", "host_covis", "host_clear"]


def scene(name):
    if name.startswith("size_"):
        return sizes(int(name[5:]))
    if name.startswith("tiny_K"):
        return tiny(int(name[6:]))
    if name.startswith("host_"):
        return host_call(name[5:])
    return {"word_threshold": word_threshold, "min_score": min_score, "narrowing": narrowing, "retain": retain,
            "best_covisible": best_covisible, "reloc_state": reloc_state, "loop_covisibles": loop_covisibles, "list_order": list_order,
            "nq_65535": nq_65535, "stream_chain": stream_chain}[name]()
