/* orb_oracle_bow_score.c -- CPU ORACLE (test infrastructure only; never linked into liborbfe.so) of ORBVocabulary::score as
 * LoopClosing::DetectLoop uses it (src/LoopClosing.cc:117-131):
 *   L1Scoring::score          Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-67
 *   the minScore loop         src/LoopClosing.cc:117-131
 * BowVectors are sorted arrays of (word id, value), as everywhere in the oracle.  Built into its own library
 * (liborb_oracle_bow_score.so) by oracle/bow_score.py with the flags of oracle/Makefile; pinned to the reference's DBoW2 by
 * tests/test_oracle_bow_score.py.  LoopClosing.cc itself needs ROS and is not compiled: its five-line loop is restated.
 */
#include <math.h>
#include <stdint.h>

double orb_oracle_bow_score(const int32_t *i1, const double *v1, int n1, const int32_t *i2, const double *v2, int n2);
float orb_oracle_loop_min_score(const int32_t *q_ids, const double *q_vals, int nq, int ncov, const int32_t *c_ptr, const int32_t *c_ids,
                                const double *c_vals, const uint8_t *bad);

/* L1Scoring::score, ScoringObject.cpp:23-67 (the lower_bound jumps restated as linear advances to the first element >= the
 * other side's id: the same element) */
double orb_oracle_bow_score(const int32_t *i1, const double *v1, int n1, const int32_t *i2, const double *v2, int n2) {
    int a = 0, b = 0;
    double score = 0;
    while (a != n1 && b != n2) {
        const double vi = v1[a], wi = v2[b];
        if (i1[a] == i2[b]) {
            score += fabs(vi - wi) - fabs(vi) - fabs(wi);
            ++a; ++b;
        } else if (i1[a] < i2[b]) {
            while (a != n1 && i1[a] < i2[b]) ++a; /* v1.lower_bound(v2_it->first) */
        } else {
            while (b != n2 && i2[b] < i1[a]) ++b;
        }
    }
    score = -score / 2.0;
    return score;
}

/* minScore of LoopClosing::DetectLoop, LoopClosing.cc:117-131: the least ORBVocabulary::score of the current keyframe's
 * BowVector against its connected keyframes, as a float starting at 1.  Connected keyframe k owns
 * c_ids/c_vals[c_ptr[k] .. c_ptr[k+1]); bad[k] != 0 is isBad() (skipped). */
float orb_oracle_loop_min_score(const int32_t *q_ids, const double *q_vals, int nq, int ncov, const int32_t *c_ptr, const int32_t *c_ids,
                                const double *c_vals, const uint8_t *bad) {
    float minScore = 1;
    for (int k = 0; k < ncov; k++) {
        if (bad[k]) continue;
        float score = orb_oracle_bow_score(q_ids, q_vals, nq, c_ids + c_ptr[k], c_vals + c_ptr[k], c_ptr[k + 1] - c_ptr[k]);
        if (score < minScore) minScore = score;
    }
    return minScore;
}
