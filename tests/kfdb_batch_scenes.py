"""Keyframe-database scenes for batches of queries (include/orbfe_bow.h orbfe_kfdb_detect_batch_device).  numpy only: op
sequences in the format of kfdb_scenarios.replay, built with kfdb_domain_scenes.Scene and its dyadic BowVectors (`kf(words,
score)`: the L1 score against a query of value QV on every word is `score`).  A batch is a maximal run of consecutive
queries of one mode (runs() below); the scenes separate the runs they mean by a host call that changes nothing (a
covisibility refresh with the same lists) or by a query of the other mode.

Every scene carries the facts it is built to produce on the sequential oracle (oracle/kfdb.py, one call per query) and the
wrong batch variants whose outcome it changes (tests/test_oracle_kfdb_batch.py runs each on a batch model):
  stale_first      a stale score read from the FIRST earlier query of the batch that scored the slot
  stale_prebatch   a stale score read from the value before the batch only
  stale_later      a stale score read that also sees later queries of the batch (the batch's last scorer)
  writeback_first  the persistent score after the batch from the first query that scored the slot
  conn_shared      one set of connected keyframes (the union) for every loop query of the batch
  firstpos_shared  one spAlreadyAddedKF for the whole batch"""
import numpy as np

import kfdb_scenarios as KS
from kfdb_domain_scenes import QV, Scene, kf

VARIANTS = ("stale_first", "stale_prebatch", "stale_later", "writeback_first", "conn_shared", "firstpos_shared")


def runs(ops):
    """The ops as a list of ("op", op) and ("run", [query ops]) items, a run being a maximal sequence of consecutive queries of
    one mode."""
    out = []
    for op in ops:
        if op[0] in ("loop", "reloc"):
            if out and out[-1][0] == "run" and out[-1][1][-1][0] == op[0]:
                out[-1][1].append(op)
            else:
                out.append(("run", [op]))
        else:
            out.append(("op", op))
    return out


def longest_run(ops):
    return max([len(r) for k, r in runs(ops) if k == "run"], default=0)


def replay_batched(db, ops, size):
    """Replay ops on anything with add / erase / clear / set_covisibles and detect_batch(mode, query ops) -> [(candidates,
    words, scores)], every run cut into batches of `size` queries (None: the whole run).  Returns every query's outputs."""
    out = []
    for kind, item in runs(ops):
        if kind == "op":
            out += KS.replay(db, [item])
            continue
        n = size or len(item)
        for i in range(0, len(item), n):
            chunk = item[i:i + n]
            out += db.detect_batch(0 if chunk[0][0] == "loop" else 1, chunk)
    return out


def _sep(s, A):
    """A host call that changes nothing: it ends the run of queries before it."""
    s.covis({A: s._lists.get(A, [])})


def _scene(name, K):
    s = Scene(name, K)
    s._lists = {}
    return s


def _covis(s, lists):
    s._lists.update(lists)
    s.covis(lists)


def _first(W, v):
    """Query values QV on every word of W but `v` on the first: a keyframe kf(W, x) with x >= v scores v."""
    vals = np.full(len(W), QV)
    vals[0] = v
    return vals


# ---- a. a stale read inside the batch: the last of two earlier scorers wins ----------------------------------------------------
def two_scorers():
    """N is A's best covisible.  Queries 0 and 1 score N (1, then 0.5); query 2 touches N with one word and reads its stale
    mRelocScore: 0.5, the last one; the first would be 1, the value before the batch 0 (candidate A)."""
    s = _scene("two_scorers", K=4)
    WA, WN = s.block(5), s.block(5)
    A, N = 0, 1
    s.add(A, *kf(WA, 0.25))
    s.add(N, *kf(WN, 1.0))
    _covis(s, {A: [N]})
    q0 = s.reloc(WN)
    q1 = s.reloc(WN, _first(WN, 0.5))
    q2 = s.reloc(WA + [WN[0]])
    s.fact(q0, "score", N, 1.0)
    s.fact(q1, "score", N, 0.5)
    s.fact(q2, "words", N, 1)
    s.fact(q2, "score", N, 0.5)
    s.cands(q2, [N])
    s.kills |= {"stale_first", "stale_prebatch"}
    return s.finish()


# ---- b. a stale read no query of the batch wrote, then a later scorer of that slot -----------------------------------------------
def prebatch_then_later():
    """N is scored 1 by a single query before the batch.  In the batch, query 1 reads it stale (1: candidate N), then query 2
    scores it 0.5: a read that saw the later query would take 0.5 (score fact)."""
    s = _scene("prebatch_then_later", K=4)
    WA, WN = s.block(5), s.block(5)
    A, N = 0, 1
    s.add(A, *kf(WA, 0.25))
    s.add(N, *kf(WN, 1.0))
    _covis(s, {A: [N]})
    s.fact(s.reloc(WN), "score", N, 1.0)
    _sep(s, A)
    q1 = s.reloc(WA + [WN[0]])
    q2 = s.reloc(WN, _first(WN, 0.5))
    s.fact(q1, "score", N, 1.0)
    s.cands(q1, [N])
    s.fact(q2, "score", N, 0.5)
    s.kills |= {"stale_later"}
    return s.finish()


# ---- c. a slot scored later in the batch is read stale earlier; the score the batch leaves ----------------------------------------
def later_scorer_and_writeback():
    """Query 0 reads N stale before queries 1 and 2 score it (1, then 0.5): it sees N's fresh 0 and returns A.  After the
    batch N holds 0.5, the last scorer's; the single query after reads it (candidate N, score 0.5)."""
    s = _scene("later_scorer_and_writeback", K=4)
    WA, WN = s.block(5), s.block(5)
    A, N = 0, 1
    s.add(A, *kf(WA, 0.25))
    s.add(N, *kf(WN, 1.0))
    _covis(s, {A: [N]})
    q0 = s.reloc(WA + [WN[0]])
    s.reloc(WN)
    s.reloc(WN, _first(WN, 0.5))
    _sep(s, A)
    q3 = s.reloc(WA + [WN[0]])
    s.fact(q0, "score", N, 0.0)
    s.cands(q0, [A])
    s.fact(q3, "score", N, 0.5)
    s.cands(q3, [N])
    s.kills |= {"stale_later", "writeback_first"}
    return s.finish()


# ---- d. the same BowVector row twice, empty rows and queries without a qualifying keyframe in between ---------------------------
def repeats_and_empties():
    """Query 0 scores N; then an empty query, a query of words no keyframe holds, two identical queries that read N stale
    (candidate N), and a last copy of query 0 with N's other score.  The identical rows give identical results."""
    s = _scene("repeats_and_empties", K=4)
    WA, WN, WX = s.block(5), s.block(5), s.block(3)
    A, N = 0, 1
    s.add(A, *kf(WA, 0.25))
    s.add(N, *kf(WN, 1.0))
    _covis(s, {A: [N]})
    s.reloc(WN, _first(WN, 0.75))
    qe = s.reloc([])
    qx = s.reloc(WX)
    qa = s.reloc(WA + [WN[0]])
    qb = s.reloc(WA + [WN[0]])
    s.reloc(WN)
    for q in (qe, qx):
        s.cands(q, [])
    for q in (qa, qb):
        s.fact(q, "score", N, 0.75)
        s.cands(q, [N])
    s.kills |= {"stale_prebatch", "stale_later"}
    return s.finish()


# ---- e. loop batches: connected sets, min scores, a keyframe two queries return -------------------------------------------------
def loop_batch():
    """Three keyframes on the same words (C 1, E 0.75, D 0.5).  Query 0 has C connected (candidate E), query 1 none (C), query
    2 E with minScore NaN (none), query 3 D with +inf (none), query 4 D with 0.6 (C: the keyframe query 1 returned too),
    query 5 C and D with -0.0 (E).  One connected set for the batch would drop C from query 1; one spAlreadyAddedKF would
    drop it from query 4."""
    s = _scene("loop_batch", K=4)
    W = s.block(6)
    C, D, E = 0, 1, 2
    s.add(C, *kf(W, 1.0))
    s.add(D, *kf(W, 0.5))
    s.add(E, *kf(W, 0.75))
    q0 = s.loop(W, conn=[C], min_score=-np.inf)
    q1 = s.loop(W, min_score=0.0)
    q2 = s.loop(W, conn=[E], min_score=np.nan)
    q3 = s.loop(W, conn=[D], min_score=np.inf)
    q4 = s.loop(W, conn=[D], min_score=0.6)
    q5 = s.loop(W, conn=[C, D], min_score=-0.0)
    s.fact(q0, "words", C, 1)
    s.cands(q0, [E])
    s.fact(q1, "words", C, 6)
    s.cands(q1, [C])
    s.cands(q2, [])
    s.cands(q3, [])
    s.fact(q4, "words", D, 1)
    s.cands(q4, [C])
    s.cands(q5, [E])
    s.kills |= {"conn_shared", "firstpos_shared"}
    return s.finish()


# ---- f. many queries of one batch return the same keyframe ----------------------------------------------------------------------
def shared_candidate(n=16):
    """n identical relocalisation rows whose one candidate is B (the best covisible of every qualifying keyframe): every query
    returns [B]; one spAlreadyAddedKF for the batch would return it once."""
    s = _scene("shared_candidate", K=8)
    W = s.block(4)
    B = 5
    for k in range(4):
        s.add(k, *kf(W, 0.5))
    s.add(B, *kf(W, 1.0))
    _covis(s, {k: [B] for k in range(4)})
    for _ in range(n):
        s.cands(s.reloc(W), [B])
    s.kills |= {"firstpos_shared"}
    return s.finish()


def all_scenes():
    return [two_scorers(), prebatch_then_later(), later_scorer_and_writeback(), repeats_and_empties(), loop_batch(), shared_candidate()]


SCENE_NAMES = ["two_scorers", "prebatch_then_later", "later_scorer_and_writeback", "repeats_and_empties", "loop_batch", "shared_candidate"]


def scene(name):
    return {"two_scorers": two_scorers, "prebatch_then_later": prebatch_then_later, "later_scorer_and_writeback": later_scorer_and_writeback,
            "repeats_and_empties": repeats_and_empties, "loop_batch": loop_batch, "shared_candidate": shared_candidate}[name]()
