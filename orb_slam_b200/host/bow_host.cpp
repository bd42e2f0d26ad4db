// bow_host.cpp -- host half of orbfe_bow_db_detect:
// KeyFrameDatabase::DetectLoopCandidates / DetectRelocalisationCandidates on arrays (include/orbfe_bow.h).
// Device: per keyframe, shared-word count + first shared word + L1 score (bow_db_score_kernel).  Host: the reference's
// list logic.  lKFsSharingWords is filled while walking the query's words in ascending order and, inside a word, the
// inverted-file list in insertion order: a keyframe enters at its FIRST shared word, so the list order is
// (first shared word, keyframe index) -- keyframe indices are insertion order by contract.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/orbfe_bow.h"
#include "../csrc/orbfe_internal.h"

extern "C" int orbfe_bow_db_detect(OrbfeMatcher *m, int mode, int nq, const int32_t *q_ids, const double *q_vals, int nkf,
                                   const int32_t *kf_ptr, const int32_t *db_ids, const double *db_vals, const uint8_t *connected,
                                   const int32_t *covis_ptr, const int32_t *covis, float min_score, int *ncand_out,
                                   int32_t *cand_out, int32_t *common_out, float *score_out) {
    if (!m || mode < 0 || mode > 1 || nq < 0 || nkf < 0 || !ncand_out) return orbfe::set_error(ORBFE_ERR_ARG, "bad arguments");
    *ncand_out = 0;
    if (nkf == 0) return ORBFE_OK;
    if (!kf_ptr || !covis_ptr || !cand_out || (nq > 0 && (!q_ids || !q_vals))) return orbfe::set_error(ORBFE_ERR_ARG, "NULL argument");
    if (kf_ptr[0] != 0 || kf_ptr[nkf] < 0 || (kf_ptr[nkf] > 0 && (!db_ids || !db_vals)) || (covis_ptr[nkf] > 0 && !covis))
        return orbfe::set_error(ORBFE_ERR_ARG, "bad CSR arrays");
    std::vector<int32_t> common(nkf), first(nkf);
    std::vector<double> score(nkf);
    const int rc = orbfe::bow_db_score(m, nq, q_ids, q_vals, nkf, kf_ptr, db_ids, db_vals, common.data(), first.data(), score.data());
    if (rc) return rc;

    const bool loop = mode == 0;
    // lKFsSharingWords (:85-104 / :206-222); connected keyframes never enter the list in loop mode
    std::vector<int> sharing;
    for (int k = 0; k < nkf; k++)
        if (common[k] > 0 && !(loop && connected && connected[k])) sharing.push_back(k);
    std::stable_sort(sharing.begin(), sharing.end(), [&](int a, int b) { return first[a] < first[b]; });
    if (common_out)
        for (int k = 0; k < nkf; k++) common_out[k] = (loop && connected && connected[k] && common[k] > 0) ? 1 : common[k];  // :92-102
    if (score_out)
        for (int k = 0; k < nkf; k++) score_out[k] = -1.0f;
    if (sharing.empty()) return ORBFE_OK;

    int maxCommonWords = 0;
    for (int k : sharing) maxCommonWords = std::max(maxCommonWords, (int)common[k]);
    const int minCommonWords = (int)((float)maxCommonWords * 0.8f);

    // scores of the keyframes with enough shared words (:124-139 / :241-252)
    std::vector<float> si(nkf, 0.f);
    std::vector<uint8_t> queried(nkf, 0), scored(nkf, 0);
    for (int k : sharing) queried[k] = 1;  // mnLoopQuery / mnRelocQuery == query id
    std::vector<std::pair<float, int>> lScoreAndMatch;
    for (int k : sharing) {
        if (common[k] > minCommonWords) {
            si[k] = (float)score[k];
            scored[k] = 1;
            if (score_out) score_out[k] = si[k];
            if (!loop || si[k] >= min_score) lScoreAndMatch.push_back({si[k], k});
        }
    }
    if (lScoreAndMatch.empty()) return ORBFE_OK;

    // accumulate by covisibility (:146-172 / :259-286)
    std::vector<std::pair<float, int>> lAcc;
    float bestAccScore = loop ? min_score : 0.f;
    for (auto &sm : lScoreAndMatch) {
        const int ki = sm.second;
        float bestScore = sm.first, accScore = sm.first;
        int best = ki;
        for (int c = covis_ptr[ki]; c < covis_ptr[ki + 1]; c++) {
            const int k2 = covis[c];
            if (k2 < 0 || k2 >= nkf) return orbfe::set_error(ORBFE_ERR_ARG, "covisibility index out of range");
            if (!queried[k2]) continue;
            // loop mode also requires mnLoopWords > minCommonWords (:157); relocalisation adds whatever mRelocScore
            // holds: a queried keyframe below the word threshold keeps the score of an earlier query -- 0 here
            if (loop && !(common[k2] > minCommonWords)) continue;
            const float s2 = scored[k2] ? si[k2] : 0.f;
            accScore += s2;
            if (s2 > bestScore) { best = k2; bestScore = s2; }
        }
        lAcc.push_back({accScore, best});
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    const float minScoreToRetain = 0.75f * bestAccScore;
    std::vector<uint8_t> added(nkf, 0);
    int nc = 0;
    for (auto &a : lAcc) {
        if (a.first > minScoreToRetain && !added[a.second]) {
            cand_out[nc++] = a.second;
            added[a.second] = 1;
        }
    }
    *ncand_out = nc;
    return ORBFE_OK;
}
