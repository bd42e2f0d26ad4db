"""The scenes of tests/kfdb_batch_scenes.py on the CPU: each one produces its facts on the sequential oracle (oracle/kfdb.py, one
call per query), the oracle equals the reference's own KeyFrameDatabase (oracle/ref_shim/ref_kfdb.cc) on it bit for bit, a
model of the batched query (per-query rows, stale reads resolved from the last earlier scorer of the batch, write-back from
the last scorer) equals the sequential oracle on every scene of kfdb_domain_scenes.py, kfdb_scenarios.py and
kfdb_batch_scenes.py whatever the batch size, and each wrong batch variant a scene names changes that scene's outcome."""
import numpy as np
import pytest

import kfdb_batch_scenes as BS
import kfdb_domain_scenes as S
import kfdb_scenarios as KS
from oracle import ref_kfdb as RK
from oracle.kfdb import F32, KeyFrameDatabase as OracleDB, l1_score

from test_oracle_kfdb import same_outputs
from test_oracle_kfdb_domain import needs_ref, voc_text  # noqa: F401  (module fixture)


class BatchModel(OracleDB):
    """detect_batch restates orbfe_kfdb_detect_batch_device on the oracle's keyframes: every query of the batch walks, scores
    and selects on its own row (words, touched list, scores it computed), a score read resolves to the last query a <= b
    of the batch that scored the slot, else the persistent score, and the persistent scores are written back after every
    query has selected.  `variant` changes one of those decisions (kfdb_batch_scenes.VARIANTS): a test device."""

    def __init__(self, K, variant=None):
        super().__init__(K)
        self.variant = variant

    def detect_batch(self, mode, qops):
        v, loop, B = self.variant, mode == 0, len(qops)
        self.qid += B
        conns = [set(int(c) for c in op[3]) if loop else set() for op in qops]
        if v == "conn_shared":
            conns = [set().union(*conns)] * B
        persistent = lambda kf: kf.loop_score if loop else kf.reloc_score
        rows = []
        for b, op in enumerate(qops):
            q_ids, q_vals = np.asarray(op[1], np.int64).tolist(), np.asarray(op[2], np.float64).tolist()
            words, touched, sharing = {}, [], []
            for w in q_ids:
                for kf in self.inv.get(w, ()):
                    if kf.slot not in words:
                        words[kf.slot] = 0
                        touched.append(kf)
                        if kf.slot not in conns[b]:
                            sharing.append(kf)
                    words[kf.slot] = 1 if kf.slot in conns[b] else words[kf.slot] + 1   # a connected one resets per visit
            min_common = int(F32(max(words[k.slot] for k in sharing)) * F32(0.8)) if sharing else 0
            scored = {kf.slot: F32(l1_score(q_ids, q_vals, kf.ids, kf.vals)) for kf in sharing if words[kf.slot] > min_common}
            rows.append((words, touched, sharing, min_common, scored, F32(op[4]) if loop else F32(0)))

        def read(b, kf):
            s = kf.slot
            if s in rows[b][4]:
                return rows[b][4][s]
            if v == "stale_prebatch":
                order = []
            elif v == "stale_first":
                order = range(b)
            elif v == "stale_later":
                order = [a for a in range(B - 1, -1, -1) if a != b]
            else:
                order = range(b - 1, -1, -1)
            for a in order:
                if s in rows[a][4]:
                    return rows[a][4][s]
            return persistent(kf)

        out, added_batch = [], set()
        for b, (words, touched, sharing, min_common, scored, min_score) in enumerate(rows):
            added = added_batch if v == "firstpos_shared" else set()
            out.append((np.array(self._select_row(loop, b, words, sharing, min_common, scored, min_score, read, added), np.int32),
                        *self._fields(words, touched, lambda kf: read(b, kf))))
        for s in set().union(*[r[4] for r in rows]):
            scorers = [a for a in range(B) if s in rows[a][4]]
            si = rows[scorers[0] if v == "writeback_first" else scorers[-1]][4][s]
            if loop:
                self.slots[s].loop_score = si
            else:
                self.slots[s].reloc_score = si
        return out

    def _fields(self, words, touched, score):
        w, sc = np.full(self.K, -1, np.int32), np.full(self.K, -1, np.float32)
        for kf in touched:
            w[kf.slot] = words[kf.slot]
            sc[kf.slot] = score(kf)
        return w, sc

    def _select_row(self, loop, b, words, sharing, min_common, scored, min_score, read, added):
        score_and_match = [(scored[kf.slot], kf) for kf in sharing if kf.slot in scored and (not loop or scored[kf.slot] >= min_score)]
        if not score_and_match:
            return []
        acc_list, best_acc = [], min_score if loop else F32(0)
        for si, kf in score_and_match:
            best_score = acc = si
            best = kf
            for kf2 in self._neighbours(kf):
                if kf2.slot not in words or (loop and kf2.slot not in scored):   # touched by this query / :158
                    continue
                s2 = read(b, kf2)
                acc = F32(acc + s2)
                if s2 > best_score:
                    best, best_score = kf2, s2
            acc_list.append((acc, best))
            if acc > best_acc:
                best_acc = acc
        retain = F32(0.75) * best_acc
        out = []
        for acc, kf in acc_list:
            if acc > retain and kf.slot not in added:
                out.append(kf.slot)
                added.add(kf.slot)
        return out


def _outcome(out):
    return [(c.tolist(), w.tolist(), s.view(np.int32).tolist()) for c, w, s in out]


def _all_scenes():
    named = [("batch/" + n, BS.scene(n)) for n in BS.SCENE_NAMES] + [("domain/" + n, S.scene(n)) for n in S.SCENE_NAMES]
    seq = []
    for seed in (1, 2, 3):
        ops, K = KS.mixed_sequence(seed)
        seq.append(("mixed/%d" % seed, ops, K))
    ops = KS.stale_reloc_sequence()
    seq.append(("stale_reloc", ops, 3))
    return [(n, sc.ops, sc.K) for n, sc in named] + seq


ALL = _all_scenes()


# ---- each batch scene hits its events ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BS.SCENE_NAMES)
def test_batch_scene_produces_its_facts(name):
    sc = BS.scene(name)
    out = KS.replay(OracleDB(sc.K), sc.ops)
    assert len(out) == sc.nq and sc.facts
    for f in sc.facts:
        kind, q = f[0], f[1]
        cands, words, scores = out[q]
        if kind == "cands":
            assert cands.tolist() == f[2], (name, f, cands.tolist())
        elif kind == "words":
            assert words[f[2]] == f[3], (name, f, words[f[2]])
        elif kind == "score":
            assert scores[f[2]].view(np.int32) == F32(f[3]).view(np.int32), (name, f, scores[f[2]])
        else:
            raise AssertionError(kind)


def test_batch_scene_shapes():
    """The scenes' batches are runs of several queries; the loop scene has connected sets and min scores of every kind."""
    for name in BS.SCENE_NAMES:
        assert BS.longest_run(BS.scene(name).ops) >= 2, name
    loop = [op for op in BS.loop_batch().ops if op[0] == "loop"]
    ms = [op[4] for op in loop]
    assert np.isnan(ms).any() and np.inf in ms and -np.inf in ms and len({tuple(op[3]) for op in loop}) >= 4
    assert BS.longest_run(BS.shared_candidate().ops) == 16


# ---- the batch model is the sequential oracle ----------------------------------------------------------------------------------
@pytest.mark.parametrize("size", [1, 2, 3, None], ids=["b1", "b2", "b3", "run"])
@pytest.mark.parametrize("name,ops,K", ALL, ids=[a[0] for a in ALL])
def test_batch_model_equals_the_sequential_oracle(name, ops, K, size):
    want = _outcome(KS.replay(OracleDB(K), ops))
    assert _outcome(BS.replay_batched(BatchModel(K), ops, size)) == want


# ---- each scene discriminates ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BS.SCENE_NAMES)
def test_batch_scene_discriminates_its_variants(name):
    sc = BS.scene(name)
    want = _outcome(KS.replay(OracleDB(sc.K), sc.ops))
    for v in sorted(sc.kills):
        assert _outcome(BS.replay_batched(BatchModel(sc.K, v), sc.ops, None)) != want, (name, v)


def test_every_batch_variant_is_discriminated():
    killed = set()
    for name in BS.SCENE_NAMES:
        killed |= BS.scene(name).kills
    assert killed == set(BS.VARIANTS)


# ---- oracle == reference ---------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("name", BS.SCENE_NAMES)
def test_oracle_equals_the_reference_on_the_batch_scene(voc_text, name):
    sc = BS.scene(name)
    same_outputs(KS.replay(OracleDB(sc.K), sc.ops), KS.replay(RK.RefKeyFrameDatabase(voc_text, sc.K), sc.ops), name)
