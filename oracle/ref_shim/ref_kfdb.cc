// oracle/ref_shim/ref_kfdb.cc -- extern "C" driver of the reference's OWN KeyFrameDatabase (src/KeyFrameDatabase.cc) for
// scripted sequences of add / erase / clear / covisibility changes / queries (TEST INFRASTRUCTURE ONLY).
//
// Built by oracle/ref_kfdb.py into oracle/_ref/libref_kfdb.so next to, and linked against, libref_orbslam.so: the
// KeyFrame / KeyFrameDatabase / DBoW2 code that runs is the reference's, compiled unmodified there.  Frames come from that
// library's ref_frame_from_arrays.  Each handle owns its vocabulary, map and database; keyframe k is the k-th add().
// Keyframes are placed in zeroed memory: KeyFrame's constructor leaves mLoopScore / mRelocScore uninitialised, and the
// reference driver's zeroed pages read 0, which is what the library defines at add.
#include <opencv2/core/core.hpp>
#include <boost/thread.hpp>
#include <cstdint>
#include <cstdlib>
#include <new>
#include <set>
#include <vector>

#include "Frame.h"
#include "KeyFrame.h"
#include "KeyFrameDatabase.h"
#include "Map.h"

using namespace ORB_SLAM;

extern "C" void *ref_frame_from_arrays(const void *kps, const uint8_t *desc, int n, int W, int H, float fx, float fy, float cx, float cy,
                                       float scale_factor, int nlevels);
extern "C" void ref_frame_free(void *f);

namespace {
struct KfDb {
    ORBVocabulary voc;
    Map map;
    KeyFrameDatabase *db;
    std::vector<KeyFrame *> kfs;
    KfDb() : db(NULL) {}
};

Frame *bare_frame() {
    return static_cast<Frame *>(ref_frame_from_arrays(NULL, NULL, 0, 64, 48, 50.f, 50.f, 32.f, 24.f, 1.2f, 8));
}

DBoW2::BowVector bow_from(const int *ids, const double *vals, int n) {
    DBoW2::BowVector v;
    for (int i = 0; i < n; i++) v.addWeight((DBoW2::WordId)ids[i], vals[i]);
    return v;
}

KeyFrame *new_keyframe(KfDb *D, const int *ids, const double *vals, int n) {
    Frame *F = bare_frame();
    void *mem = std::calloc(1, sizeof(KeyFrame));
    KeyFrame *kf = new (mem) KeyFrame(*F, &D->map, D->db);
    ref_frame_free(F);
    kf->mBowVec = bow_from(ids, vals, n);
    return kf;
}

int index_of(KfDb *D, KeyFrame *kf) {
    for (size_t k = 0; k < D->kfs.size(); k++)
        if (D->kfs[k] == kf) return (int)k;
    return -1;
}

int copy_out(KfDb *D, const std::vector<KeyFrame *> &c, int *out, int cap) {
    for (size_t i = 0; i < c.size() && (int)i < cap; i++) out[i] = index_of(D, c[i]);
    return (int)c.size();
}
}  // namespace

extern "C" {

void *ref_kfdb_create(const char *voc_text) {
    KfDb *D = new KfDb();
    if (!D->voc.loadFromTextFile(voc_text)) { delete D; return NULL; }
    D->db = new KeyFrameDatabase(D->voc);
    return D;
}

// KeyFrameDatabase::add (:39-45) of a new keyframe with the given BowVector; returns its index
int ref_kfdb_add(void *h, const int *ids, const double *vals, int n) {
    KfDb *D = static_cast<KfDb *>(h);
    KeyFrame *kf = new_keyframe(D, ids, vals, n);
    D->db->add(kf);
    D->kfs.push_back(kf);
    return (int)D->kfs.size() - 1;
}

// KeyFrameDatabase::erase (:47-66); the keyframe object stays, as a bad keyframe's does
void ref_kfdb_erase(void *h, int k) {
    KfDb *D = static_cast<KfDb *>(h);
    D->db->erase(D->kfs[k]);
}

// KeyFrameDatabase::clear (:68-72)
void ref_kfdb_clear(void *h) { static_cast<KfDb *>(h)->db->clear(); }

// replace the connections of keyframe k: GetBestCovisibilityKeyFrames(10) then returns `others` in this order
void ref_kfdb_set_covisibles(void *h, int k, const int *others, int n) {
    KfDb *D = static_cast<KfDb *>(h);
    KeyFrame *kf = D->kfs[k];
    const std::set<KeyFrame *> old = kf->GetConnectedKeyFrames();
    for (std::set<KeyFrame *>::const_iterator it = old.begin(); it != old.end(); ++it) kf->EraseConnection(*it);
    for (int i = 0; i < n; i++) kf->AddConnection(D->kfs[others[i]], 1000 - i);
}

// DetectLoopCandidates(pKF, minScore) (:75-196) for a fresh query keyframe connected to `connected`
int ref_kfdb_detect_loop(void *h, const int *q_ids, const double *q_vals, int nq, const int *connected, int nconn, float min_score,
                         int *out, int cap) {
    KfDb *D = static_cast<KfDb *>(h);
    KeyFrame *q = new_keyframe(D, q_ids, q_vals, nq);
    for (int i = 0; i < nconn; i++) q->AddConnection(D->kfs[connected[i]], 100);
    return copy_out(D, D->db->DetectLoopCandidates(q, min_score), out, cap);
}

// DetectRelocalisationCandidates(Frame *F) (:198-308)
int ref_kfdb_detect_reloc(void *h, const int *q_ids, const double *q_vals, int nq, int *out, int cap) {
    KfDb *D = static_cast<KfDb *>(h);
    Frame *F = bare_frame();
    F->mBowVec = bow_from(q_ids, q_vals, nq);
    const int n = copy_out(D, D->db->DetectRelocalisationCandidates(F), out, cap);
    ref_frame_free(F);
    return n;
}

}  // extern "C"
