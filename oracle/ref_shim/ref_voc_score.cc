// oracle/ref_shim/ref_voc_score.cc -- extern "C" driver of the reference's OWN ORBVocabulary::score (DBoW2
// TemplatedVocabulary::score -> L1Scoring::score), the call of LoopClosing.cc:127 (TEST INFRASTRUCTURE ONLY).
//
// Built by oracle/Makefile into oracle/_ref/libref_drivers.so next to, and linked against, libref_orbslam.so: the
// DBoW2 code that runs is the reference's, compiled unmodified there.  A handle owns a vocabulary loaded from DBoW2's text
// format; its header names the scoring object.
#include <opencv2/core/core.hpp>

#include "ORBVocabulary.h"

using namespace ORB_SLAM;

namespace {
DBoW2::BowVector bow_from(const int *ids, const double *vals, int n) {
    DBoW2::BowVector v;
    for (int i = 0; i < n; i++) v.addWeight((DBoW2::WordId)ids[i], vals[i]);
    return v;
}
}  // namespace

extern "C" {

void *ref_voc_score_create(const char *voc_text) {
    ORBVocabulary *voc = new ORBVocabulary();
    if (!voc->loadFromTextFile(voc_text)) { delete voc; return NULL; }
    return voc;
}

void ref_voc_score_free(void *h) { delete static_cast<ORBVocabulary *>(h); }

// mpORBVocabulary->score(v1, v2)
double ref_voc_score(void *h, const int *ids1, const double *vals1, int n1, const int *ids2, const double *vals2, int n2) {
    return static_cast<ORBVocabulary *>(h)->score(bow_from(ids1, vals1, n1), bow_from(ids2, vals2, n2));
}

}  // extern "C"
