"""The scenes of tests/kfdb_domain_scenes.py on the CPU: each one produces the facts it is built for (on the stateful oracle,
oracle/kfdb.py), its outcome changes under the plausible wrong variants it is built against, and on it the oracle equals the
reference's own KeyFrameDatabase (oracle/_ref, driven by oracle/ref_shim/ref_kfdb.cc) bit for bit: candidates, words and
scores."""
import os

import numpy as np
import pytest

import kfdb_domain_scenes as S
import kfdb_scenarios as KS
from oracle import ref as R
from oracle import ref_kfdb as RK
from oracle.kfdb import F32, KeyFrameDatabase as OracleDB, l1_score

from test_oracle_kfdb import same_outputs

HAVE_REF = RK.available() or os.path.isdir(os.path.join(R.REFERENCE_ROOT, "src"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libref_drivers.so not built and the reference sources are absent")


def run_oracle(sc):
    return KS.replay(OracleDB(sc.K), sc.ops)


def _queries(sc):
    return [op for op in sc.ops if op[0] in ("loop", "reloc")]


# ---- each scene hits its events -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", S.SCENE_NAMES)
def test_scene_produces_its_facts(name):
    sc = S.scene(name)
    out = run_oracle(sc)
    qops = _queries(sc)
    assert len(out) == sc.nq and sc.facts
    for f in sc.facts:
        kind, q = f[0], f[1]
        cands, words, scores = out[q]
        if kind == "cands":
            assert cands.tolist() == f[2], (name, f, cands.tolist()[:20])
        elif kind == "words":
            assert words[f[2]] == f[3], (name, f, words[f[2]])
        elif kind == "score":
            assert scores[f[2]].view(np.int32) == F32(f[3]).view(np.int32), (name, f, scores[f[2]])
        elif kind == "min_common":
            conn = set(qops[q][3]) if qops[q][0] == "loop" else set()
            touched = [s for s in np.flatnonzero(words >= 0) if s not in conn]
            assert int(F32(max(words[touched])) * F32(0.8)) == f[2], (name, f)
        else:
            raise AssertionError(kind)


def test_scene_shapes():
    """The sizes straddle the 1024-entry chunks; the order scene compacts the store between its queries; nq 65535 is used."""
    for n in (1023, 1024, 1025, 2049, 5000):
        sc = S.sizes(n)
        assert sc.K & (sc.K - 1) and len(run_oracle(sc)[0][0]) > min(n // 2, 1024)
    assert S.list_order().compactions >= 1
    assert max(len(op[1]) for op in _queries(S.nq_65535())) == 65535
    e = [f for f in S.best_covisible().facts if f[0] == "cands"]
    assert all(len(f[2]) == 2 for f in e[-2:])


# ---- each scene discriminates -------------------------------------------------------------------------------------------------
class VariantDB(OracleDB):
    """The oracle with one decision of _select (or the order of its sharing list) changed: a test device, not an oracle."""

    def __init__(self, K, variant):
        super().__init__(K)
        self.variant, self.seq, self._seq = variant, 0, {}

    def add(self, slot, ids, vals):
        super().add(slot, ids, vals)
        self.seq += 1
        self._seq[id(self.slots[slot])] = self.seq

    def _select(self, loop, qid, sharing, q_ids, q_vals, min_score):
        v = self.variant
        if not sharing:
            return []
        first = lambda ks: next(i for i, w in enumerate(q_ids) if w in ks)
        if v == "order_slot":
            sharing = sorted(sharing, key=lambda k: k.slot)
        elif v == "order_add":
            sharing = sorted(sharing, key=lambda k: self._seq[id(k)])
        elif v == "order_word":
            sharing = sorted(sharing, key=lambda k: (first(set(k.ids)), k.slot))
        gt = lambda a, b, ge: a >= b if ge else a > b
        nwords = (lambda k: k.loop_words) if loop else (lambda k: k.reloc_words)
        max_common = max(nwords(k) for k in sharing)
        min_common = int(F32(max_common) * F32(0.8))

        def narrow(d):
            if v == "no_narrow":
                return np.float64(d)
            f = F32(d)
            if v == "narrow_rz" and abs(float(f)) > abs(d):
                f = np.nextafter(f, F32(0))
            return f

        fresh, score_and_match = set(), []
        for kf in sharing:
            if gt(nwords(kf), min_common, v == "words_ge"):
                si = narrow(l1_score(q_ids, q_vals, kf.ids, kf.vals))
                fresh.add(id(kf))
                if loop:
                    kf.loop_score = si
                    if (si > min_score) if v == "minscore_gt" else (si >= min_score):
                        score_and_match.append((si, kf))
                else:
                    kf.reloc_score = si
                    score_and_match.append((si, kf))
        if not score_and_match:
            return []
        acc_list = []
        best_acc = min_score if loop else F32(0)
        for si, kf in score_and_match:
            best_score = si
            best = kf
            terms = []
            for kf2 in self._neighbours(kf):
                if loop:
                    if kf2.loop_query != qid or not gt(kf2.loop_words, min_common, v == "words_ge"):
                        continue
                    s2 = kf2.loop_score
                else:
                    if kf2.reloc_query != qid:
                        continue
                    s2 = kf2.reloc_score if (v != "stale_zero" or id(kf2) in fresh) else F32(0)
                terms.append(s2)
                if gt(s2, best_score, v == "best_ge"):
                    best, best_score = kf2, s2
            if v == "acc_double":
                acc = F32(float(si) + sum(float(t) for t in terms))
            else:
                acc = si
                for t in (terms[::-1] if v == "acc_reversed" else terms):
                    acc = acc + t if v == "no_narrow" else F32(acc + t)
            acc_list.append((acc, best))
            if acc > best_acc:
                best_acc = acc
        retain = F32(0.75) * best_acc
        out, added = [], set()
        for acc, kf in acc_list:
            if gt(acc, retain, v == "retain_ge") and id(kf) not in added:
                out.append(kf.slot)
                added.add(id(kf))
        return out


def _outcome(db, sc):
    return [(c.tolist(), w.tolist(), s.view(np.int32).tolist()) for c, w, s in KS.replay(db, sc.ops)]


@pytest.mark.parametrize("name", S.SCENE_NAMES)
def test_scene_discriminates_its_variants(name):
    sc = S.scene(name)
    want = _outcome(OracleDB(sc.K), sc)
    assert _outcome(VariantDB(sc.K, None), sc) == want      # the restatement without a change is the oracle
    for v in sorted(sc.kills):
        assert _outcome(VariantDB(sc.K, v), sc) != want, (name, v)


def test_every_variant_is_discriminated():
    killed = set()
    for name in S.SCENE_NAMES:
        killed |= S.scene(name).kills
    assert killed == set(S.VARIANTS)


# ---- oracle == reference ------------------------------------------------------------------------------------------------------
def vocabulary_text(path, k=16, L=4):
    """A complete k-ary tree of depth L in DBoW2's text format: k^L words (65536 for 16, 4), word id = leaf order."""
    first_leaf = sum(k ** l for l in range(L))
    n_nodes = first_leaf + k ** L
    with open(path, "w") as f:
        f.write("%d %d 0 0\n" % (k, L))
        f.write("\n".join("%d %d %s 1.0" % ((nid - 1) // k, 1 if nid >= first_leaf else 0, " ".join(["0"] * 32)) for nid in range(1, n_nodes)))


@pytest.fixture(scope="module")
def voc_text(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("kfdb_domain") / "voc16x4.txt")
    vocabulary_text(path)
    return path


@needs_ref
@pytest.mark.parametrize("name", S.SCENE_NAMES)
def test_oracle_equals_the_reference_on_the_scene(voc_text, name):
    sc = S.scene(name)
    same_outputs(run_oracle(sc), KS.replay(RK.RefKeyFrameDatabase(voc_text, sc.K), sc.ops), name)
