"""Stateful oracle of KeyFrameDatabase (reference src/KeyFrameDatabase.cc:39-308) together with the six KeyFrame query fields
(mnLoopQuery, mnLoopWords, mLoopScore, mnRelocQuery, mnRelocWords, mRelocScore; KeyFrame.h:160-165), restated in Python
on the slot interface of orbfe_kfdb_* (include/orbfe_bow.h).  Float arithmetic is float32 where the reference's is float
(numpy scalars), the L1 score is summed in double in ascending word order and narrowed to float.

Slots: a keyframe is added into a slot and erased from it; a covisibility entry names a slot and reads whatever keyframe
is in it at query time (an empty slot contributes nothing).  Query ids are one counter over both modes, as the library's."""
import numpy as np

F32 = np.float32


class _KeyFrame:
    __slots__ = ("slot", "ids", "vals", "loop_query", "loop_words", "loop_score", "reloc_query", "reloc_words", "reloc_score")

    def __init__(self, slot, ids, vals):
        self.slot = slot
        self.ids, self.vals = np.asarray(ids, np.int64).tolist(), np.asarray(vals, np.float64).tolist()
        # a fresh KeyFrame: stamps 0 (KeyFrame.cc:33); the scores are 0 (the library defines them so at add)
        self.loop_query = self.reloc_query = 0
        self.loop_words = self.reloc_words = 0
        self.loop_score = self.reloc_score = F32(0)


def l1_score(q_ids, q_vals, ids, vals):
    """L1Scoring::score (ScoringObject.cpp:23-67): shared words in ascending order, double, then -score / 2."""
    a = b = 0
    score = 0.0
    while a < len(q_ids) and b < len(ids):
        if q_ids[a] == ids[b]:
            vi, wi = q_vals[a], vals[b]
            score += abs(vi - wi) - abs(vi) - abs(wi)
            a += 1
            b += 1
        elif q_ids[a] < ids[b]:
            a += 1
        else:
            b += 1
    return -score / 2.0


class KeyFrameDatabase:
    def __init__(self, max_keyframes):
        self.K = max_keyframes
        self.inv = {}                    # mvInvertedFile: word -> [keyframe, ...] in push_back order
        self.slots = [None] * max_keyframes
        self.covis = [[] for _ in range(max_keyframes)]
        self.qid = 0

    def add(self, slot, ids, vals):     # :39-45
        assert self.slots[slot] is None
        kf = _KeyFrame(slot, ids, vals)
        self.slots[slot] = kf
        for w in kf.ids:
            self.inv.setdefault(w, []).append(kf)

    def erase(self, slot):               # :47-66
        kf = self.slots[slot]
        if kf is None:
            return
        for w in kf.ids:
            lst = self.inv[w]
            for i, x in enumerate(lst):
                if x is kf:
                    del lst[i]
                    break
        self.slots[slot] = None
        self.covis[slot] = []

    def clear(self):                     # :68-72
        self.inv = {}
        self.slots = [None] * self.K
        self.covis = [[] for _ in range(self.K)]

    def set_covisibles(self, lists):
        for s, lst in lists.items():
            assert len(lst) <= 10
            self.covis[s] = [int(x) for x in lst]

    def _neighbours(self, kf):
        """GetBestCovisibilityKeyFrames(10) of kf, as the keyframes now in those slots."""
        return [self.slots[s] for s in self.covis[kf.slot] if self.slots[s] is not None]

    def detect(self, mode, q_ids, q_vals, connected=(), min_score=0.0):
        """Returns (candidate slots, words[K], scores[K]) -- the last two hold the query fields of every keyframe this query
        touched, -1 elsewhere (what orbfe_kfdb_detect writes to words_out / score_out)."""
        self.qid += 1
        qid = self.qid
        q_ids, q_vals = np.asarray(q_ids, np.int64).tolist(), np.asarray(q_vals, np.float64).tolist()
        loop = mode == 0
        min_score = F32(min_score)
        conn = set(int(c) for c in connected) if loop else set()
        sharing, touched = [], []
        seen = set()
        for w in q_ids:                                            # :85-103 / :206-221
            for kf in self.inv.get(w, ()):
                if id(kf) not in seen:
                    seen.add(id(kf))
                    touched.append(kf)
                if loop:
                    if kf.loop_query != qid:
                        kf.loop_words = 0
                        if kf.slot not in conn:
                            kf.loop_query = qid
                            sharing.append(kf)
                    kf.loop_words += 1
                else:
                    if kf.reloc_query != qid:
                        kf.reloc_words = 0
                        kf.reloc_query = qid
                        sharing.append(kf)
                    kf.reloc_words += 1
        cands = self._select(loop, qid, sharing, q_ids, q_vals, min_score)
        words, scores = np.full(self.K, -1, np.int32), np.full(self.K, -1, np.float32)
        for kf in touched:
            words[kf.slot] = kf.loop_words if loop else kf.reloc_words
            scores[kf.slot] = kf.loop_score if loop else kf.reloc_score
        return np.array(cands, np.int32), words, scores

    def _select(self, loop, qid, sharing, q_ids, q_vals, min_score):
        if not sharing:
            return []
        nwords = (lambda k: k.loop_words) if loop else (lambda k: k.reloc_words)
        max_common = max(nwords(k) for k in sharing)
        min_common = int(F32(max_common) * F32(0.8))               # int minCommonWords = maxCommonWords*0.8f
        score_and_match = []
        for kf in sharing:                                         # :124-138 / :241-252
            if nwords(kf) > min_common:
                si = F32(l1_score(q_ids, q_vals, kf.ids, kf.vals))
                if loop:
                    kf.loop_score = si
                    if si >= min_score:
                        score_and_match.append((si, kf))
                else:
                    kf.reloc_score = si
                    score_and_match.append((si, kf))
        if not score_and_match:
            return []
        acc_list = []
        best_acc = min_score if loop else F32(0)
        for si, kf in score_and_match:                             # :147-172 / :261-286
            best_score = acc = si
            best = kf
            for kf2 in self._neighbours(kf):
                if loop:
                    if kf2.loop_query != qid or not kf2.loop_words > min_common:
                        continue
                    s2 = kf2.loop_score
                else:
                    if kf2.reloc_query != qid:
                        continue
                    s2 = kf2.reloc_score                           # may be an earlier query's
                acc = F32(acc + s2)
                if s2 > best_score:
                    best, best_score = kf2, s2
            acc_list.append((acc, best))
            if acc > best_acc:
                best_acc = acc
        retain = F32(0.75) * best_acc
        out, added = [], set()
        for acc, kf in acc_list:
            if acc > retain and id(kf) not in added:
                out.append(kf.slot)
                added.add(id(kf))
        return out
