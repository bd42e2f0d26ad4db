// bow_l1.cuh -- the DBoW2 L1 score of two BowVectors on the device, shared by every kernel that scores keyframes against a
// query (bow_db_score_kernel in bow_kernels.cu, the resident keyframe database in kfdb.cu), so that both compute the
// same double-precision sum.
#pragma once

namespace orbfe {

// Two-pointer walk over the (ascending) word lists of the query q_ids/q_vals[0, nq) and of a keyframe ids/vals[b, be).
// score accumulates |vi - wi| - |vi| - |wi| over the shared words in ascending word order, as L1Scoring::score does
// (ScoringObject.cpp:33-56; its lower_bound jumps visit the same shared words in the same order), and returns -sum / 2.
// common = number of shared words, first = the first shared word id (-1 if none).
__device__ __forceinline__ double bow_l1_walk(int nq, const int *__restrict__ q_ids, const double *__restrict__ q_vals, int b0, int be0,
                                             const int *__restrict__ ids, const double *__restrict__ vals, int &common, int &first) {
    int a = 0, b = b0;
    const int be = be0;
    int c = 0, f = -1;
    double score = 0.0;
    while (a < nq && b < be) {
        const int ia = __ldg(&q_ids[a]), ib = __ldg(&ids[b]);
        if (ia == ib) {
            const double vi = __ldg(&q_vals[a]), wi = __ldg(&vals[b]);
            score = __dadd_rn(score, __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi)));
            if (c == 0) f = ia;
            c++;
            a++; b++;
        } else if (ia < ib) {
            a++;
        } else {
            b++;
        }
    }
    common = c;
    first = f;
    return -score / 2.0;
}

}  // namespace orbfe
