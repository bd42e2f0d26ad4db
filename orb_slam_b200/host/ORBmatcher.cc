// ORBmatcher.cc -- facade of ORB_SLAM::ORBmatcher (reference src/ORBmatcher.cc) over liborbfe.so.
//
// Pattern of every routine here: (1) convert -- the Frame / KeyFrame becomes an OrbfeFrameView and the map points
// become arrays (or, for the KeyFrame-level routines, projected query windows), in the reference's order;
// (2) one array-level entry of include/orbfe_match.h finds the candidates and runs the accept loop on the GPU;
// (3) replay -- the resulting matches are written back into the map, with the reference's map changes.
//
// All thirteen search / fuse methods of the reference class are defined here; every array-level entry they call has
// oracle parity tests (tests/test_gpu_matchers.py).
#include "ORBmatcher.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>

#include "orbfe.h"
#include "orbfe_match.h"

namespace ORB_SLAM {

const int ORBmatcher::TH_HIGH = 100;
const int ORBmatcher::TH_LOW = 50;
const int ORBmatcher::HISTO_LENGTH = 30;

namespace {

int g_match_device = 0;

// Error policy.  The reference's matchers cannot fail, liborbfe's calls can (a transient cudaMalloc failure in a
// scratch regrow, a launch error, an unsupported geometry).  Every failure goes through one handler: the default
// logs the code and message and the calling method returns 0 matches with the map untouched, so that a SLAM node
// survives a transient device error (Tracking treats 0 matches as a lost frame); ORBFE_ABORT_ON_ERROR=1 or
// ORBmatcher::SetErrorHandler() select another policy (e.g. abort, as round 1 did unconditionally).
void default_error_handler(int code, const char *msg) {
    std::fprintf(stderr, "ORBmatcher: liborbfe error %d: %s (there is no CPU path; returning 0 matches)\n", code, msg);
    const char *e = std::getenv("ORBFE_ABORT_ON_ERROR");
    if (e && *e && *e != '0') std::abort();
}
ORBmatcher::ErrorHandler g_error_handler = default_error_handler;

// ORBmatcher objects are stack temporaries used from three threads (Tracking.cc:352,488,556,...):
// each calling thread lazily gets its own device handle (stream + scratch buffers), destroyed when the thread exits.
struct ThreadMatcher {
    OrbfeMatcher *m;
    ThreadMatcher() : m(NULL) {}
    ~ThreadMatcher() { if (m) orbfe_matcher_destroy(m); }
};
OrbfeMatcher *thread_matcher() {
    static thread_local ThreadMatcher holder;
    if (!holder.m) {
        const int rc = orbfe_matcher_create(g_match_device, &holder.m);
        if (rc != ORBFE_OK) { holder.m = NULL; g_error_handler(rc, orbfe_last_error()); }
    }
    return holder.m;  // NULL after a failed create: the C-ABI call then reports ORBFE_ERR_ARG and the method returns 0
}

// true if the call succeeded; otherwise reports through the handler (which may abort) and returns false
bool ok(int rc) {
    if (rc == ORBFE_OK) return true;
    g_error_handler(rc, orbfe_last_error());
    return false;
}

// contiguous view of a descriptor matrix (cv::Mat rows may be strided).  Holds a reference on the Mat's buffer: KeyFrame::
// GetDescriptors() returns a CLONE (KeyFrame.cc), i.e. a temporary whose storage would otherwise die with the full expression
// -- found by tests/test_gpu_facade_vs_ref.py, which runs this file against the reference's real KeyFrame.cc.
struct DescBuf {
    cv::Mat keep;
    std::vector<unsigned char> own;
    const unsigned char *ptr;
    explicit DescBuf(const cv::Mat &d) : keep(d), ptr(NULL) {
        if (d.empty()) return;
        if (d.isContinuous()) { ptr = keep.ptr(0); return; }
        own.resize((size_t)d.rows * 32);
        for (int i = 0; i < d.rows; i++) std::memcpy(&own[(size_t)i * 32], d.ptr(i), 32);
        ptr = &own[0];
    }
};

OrbfeFrameView make_view(const Frame &F, const DescBuf &d) {
    static_assert(sizeof(cv::KeyPoint) == sizeof(OrbfeKeyPoint), "cv::KeyPoint must be the 28-byte OpenCV 2.4 layout");
    OrbfeFrameView v;
    v.n = (int)F.mvKeysUn.size();
    v.keys_un = v.n ? reinterpret_cast<const OrbfeKeyPoint *>(&F.mvKeysUn[0]) : NULL;
    v.desc = d.ptr;
    v.min_x = (float)Frame::mnMinX; v.min_y = (float)Frame::mnMinY;
    v.max_x = (float)Frame::mnMaxX; v.max_y = (float)Frame::mnMaxY;
    v.grid_inv_w = Frame::mfGridElementWidthInv;
    v.grid_inv_h = Frame::mfGridElementHeightInv;
    v.nlevels = F.mnScaleLevels;
    v.scale_factors = F.mvScaleFactors.empty() ? NULL : &F.mvScaleFactors[0];
    return v;
}

}  // namespace

ORBmatcher::ORBmatcher(float nnratio, bool checkOri) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}

void ORBmatcher::SetErrorHandler(ErrorHandler h) { g_error_handler = h ? h : default_error_handler; }

// A single pair is 8 XOR+popcount on the host: shipping 64 bytes to the GPU for one distance would only add
// latency.  Every *batched* distance computation below goes to the device.
int ORBmatcher::DescriptorDistance(const cv::Mat &a, const cv::Mat &b)
{
    const unsigned char *pa = a.ptr(0), *pb = b.ptr(0);
    int dist = 0;
    for (int i = 0; i < 32; i += 8) {
        unsigned long long x, y;
        std::memcpy(&x, pa + i, 8);
        std::memcpy(&y, pb + i, 8);
        dist += __builtin_popcountll(x ^ y);
    }
    return dist;
}

float ORBmatcher::RadiusByViewingCos(const float &viewCos) { return viewCos > 0.998 ? 2.5f : 4.0f; }  // :127-133

void ORBmatcher::ComputeThreeMaxima(std::vector<int> *histo, const int L, int &ind1, int &ind2, int &ind3)
{
    int max1 = 0, max2 = 0, max3 = 0;
    for (int i = 0; i < L; i++) {
        const int s = (int)histo[i].size();
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if (max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if (max3 < 0.1f * (float)max1) { ind3 = -1; }
}

// ---- Tracking::TrackWithMotionModel (Tracking.cc:565) -------------------------------------------------
int ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, float th)
{
    const DescBuf dc(CurrentFrame.mDescriptors), dl(LastFrame.mDescriptors);
    const OrbfeFrameView cur = make_view(CurrentFrame, dc), last = make_view(LastFrame, dl);
    const int nl = last.n, nc = cur.n;
    std::vector<unsigned char> has(nl, 0), outl(nl, 0);
    std::vector<float> world((size_t)nl * 3, 0.f);
    for (int i = 0; i < nl; i++) {
        MapPoint *pMP = LastFrame.mvpMapPoints[i];
        if (!pMP) continue;
        has[i] = 1;
        outl[i] = LastFrame.mvbOutlier[i] ? 1 : 0;
        const cv::Mat X = pMP->GetWorldPos();
        for (int k = 0; k < 3; k++) world[(size_t)i * 3 + k] = X.at<float>(k, 0);
    }
    float T[12];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) T[4 * r + c] = CurrentFrame.mTcw.at<float>(r, c);
    std::vector<int> mp(nc, -1);
    for (int i = 0; i < nc; i++)
        if (CurrentFrame.mvpMapPoints[i]) mp[i] = INT_MAX;  // already occupied slot (:1562)
    const unsigned char *hp = nl ? &has[0] : NULL, *op = nl ? &outl[0] : NULL;
    const float *wp = nl ? &world[0] : NULL, *tp = T;
    int *mpp = nc ? &mp[0] : NULL;
    int nmatches = 0;
    if (!ok(orbfe_search_by_projection_frames(thread_matcher(), 1, &cur, &last, &hp, &op, &wp, &tp, Frame::fx, Frame::fy,
                                            Frame::cx, Frame::cy, th, mbCheckOrientation ? 1 : 0, &mpp, &nmatches))) return 0;
    for (int i = 0; i < nc; i++)
        if (mp[i] >= 0 && mp[i] != INT_MAX) CurrentFrame.mvpMapPoints[i] = LastFrame.mvpMapPoints[mp[i]];
    return nmatches;
}

// ---- Tracking::TrackPreviousFrame (Tracking.cc:497-502) ------------------------------------------------
int ORBmatcher::WindowSearch(Frame &F1, Frame &F2, int windowSize, std::vector<MapPoint *> &vpMapPointMatches2,
                             int minScaleLevel, int maxScaleLevel)
{
    const DescBuf d1(F1.mDescriptors), d2(F2.mDescriptors);
    const OrbfeFrameView v1 = make_view(F1, d1), v2 = make_view(F2, d2);
    std::vector<unsigned char> has(v1.n, 0);
    for (int i = 0; i < v1.n; i++) {
        MapPoint *p = F1.mvpMapPoints[i];
        has[i] = (p && !p->isBad()) ? 1 : 0;  // :425-428
    }
    std::vector<int> m21(v2.n > 0 ? v2.n : 1, -1);
    int nmatches = 0;
    if (!ok(orbfe_window_search(thread_matcher(), &v1, &v2, v1.n ? &has[0] : NULL, windowSize, minScaleLevel, maxScaleLevel,
                              mfNNratio, mbCheckOrientation ? 1 : 0, &m21[0], &nmatches))) return 0;
    vpMapPointMatches2 = std::vector<MapPoint *>(F2.mvpMapPoints.size(), static_cast<MapPoint *>(NULL));  // :412
    for (int i2 = 0; i2 < v2.n; i2++)
        if (m21[i2] >= 0) vpMapPointMatches2[i2] = F1.mvpMapPoints[m21[i2]];
    return nmatches;
}

// ---- Tracking::Initialize (Tracking.cc:352-353) ----------------------------------------------------------
int ORBmatcher::SearchForInitialization(Frame &F1, Frame &F2, std::vector<cv::Point2f> &vbPrevMatched,
                                        std::vector<int> &vnMatches12, int windowSize)
{
    const DescBuf d1(F1.mDescriptors), d2(F2.mDescriptors);
    const OrbfeFrameView v1 = make_view(F1, d1), v2 = make_view(F2, d2);
    static_assert(sizeof(cv::Point2f) == 8, "cv::Point2f must be two packed floats");
    vnMatches12 = std::vector<int>(F1.mvKeysUn.size(), -1);  // :601
    int nmatches = 0;
    if (v1.n == 0) return 0;
    if (!ok(orbfe_search_for_initialization(thread_matcher(), &v1, &v2, reinterpret_cast<float *>(&vbPrevMatched[0]), windowSize,
                                          mfNNratio, mbCheckOrientation ? 1 : 0, &vnMatches12[0], &nmatches))) return 0;
    return nmatches;
}

// ---- Tracking::SearchReferencePointsInFrustum (Tracking.cc:724) -----------------------------------------
int ORBmatcher::SearchByProjection(Frame &F, const std::vector<MapPoint *> &vpMapPoints, const float th)
{
    const DescBuf df(F.mDescriptors);
    const OrbfeFrameView fv = make_view(F, df);
    const int np = (int)vpMapPoints.size();
    std::vector<unsigned char> in_view(np, 0), desc((size_t)np * 32 + 1, 0);
    std::vector<float> proj((size_t)np * 2 + 1, 0.f), vcos(np + 1, 0.f);
    std::vector<int> level(np + 1, 0);
    for (int i = 0; i < np; i++) {
        MapPoint *pMP = vpMapPoints[i];
        if (!pMP->mbTrackInView || pMP->isBad()) continue;  // :57-61
        in_view[i] = 1;
        proj[2 * i] = pMP->mTrackProjX; proj[2 * i + 1] = pMP->mTrackProjY;
        level[i] = pMP->mnTrackScaleLevel;
        vcos[i] = pMP->mTrackViewCos;
        const cv::Mat d = pMP->GetDescriptor();
        std::memcpy(&desc[(size_t)i * 32], d.ptr(0), 32);
    }
    std::vector<int> mp(fv.n > 0 ? fv.n : 1, -1);
    for (int i = 0; i < fv.n; i++)
        if (F.mvpMapPoints[i]) mp[i] = INT_MAX;
    int nmatches = 0;
    if (!ok(orbfe_search_local_points(thread_matcher(), &fv, np, np ? &in_view[0] : NULL, &proj[0], &level[0], &vcos[0], &desc[0], th,
                                    mfNNratio, &mp[0], &nmatches))) return 0;
    for (int i = 0; i < fv.n; i++)
        if (mp[i] >= 0 && mp[i] != INT_MAX) F.mvpMapPoints[i] = vpMapPoints[mp[i]];
    return nmatches;
}

// ---- Tracking::TrackPreviousFrame refinement (Tracking.cc:528-531) --------------------------------------
int ORBmatcher::SearchByProjection(Frame &F1, Frame &F2, int windowSize, std::vector<MapPoint *> &vpMapPointMatches2)
{
    vpMapPointMatches2 = F2.mvpMapPoints;  // :521
    const std::set<MapPoint *> found(vpMapPointMatches2.begin(), vpMapPointMatches2.end());
    const DescBuf d1(F1.mDescriptors), d2(F2.mDescriptors);
    const OrbfeFrameView v1 = make_view(F1, d1), v2 = make_view(F2, d2);
    std::vector<unsigned char> valid(v1.n + 1, 0);
    std::vector<float> world((size_t)v1.n * 3 + 1, 0.f);
    for (int i1 = 0; i1 < v1.n; i1++) {
        MapPoint *p = F1.mvpMapPoints[i1];
        if (!p || p->isBad() || found.count(p)) continue;  // :533-537
        valid[i1] = 1;
        const cv::Mat X = p->GetWorldPos();
        for (int k = 0; k < 3; k++) world[(size_t)i1 * 3 + k] = X.at<float>(k, 0);
    }
    float T[12];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) T[4 * r + c] = F2.mTcw.at<float>(r, c);
    std::vector<int> mp(v2.n > 0 ? v2.n : 1, -1);
    for (int i = 0; i < v2.n; i++)
        if (vpMapPointMatches2[i]) mp[i] = INT_MAX;
    int nmatches = 0;
    if (!ok(orbfe_search_by_projection_f1f2(thread_matcher(), &v1, &v2, &valid[0], &world[0], T, Frame::fx, Frame::fy, Frame::cx,
                                          Frame::cy, windowSize, mfNNratio, &mp[0], &nmatches))) return 0;
    for (int i = 0; i < v2.n; i++)
        if (mp[i] >= 0 && mp[i] != INT_MAX) vpMapPointMatches2[i] = F1.mvpMapPoints[mp[i]];
    return nmatches;
}

}  // namespace ORB_SLAM

// =================================================================================================
// KeyFrame-level routines.  Each projects its map points into one query window apiece, in the reference's order:
// (u, v, th * scale factor of the predicted level, levels [lv - 1, lv], the point's descriptor).  One array-level entry
// walks the KeyFrame's grid and takes the best candidate: orbfe_guided_search for SearchByProjection(KeyFrame*, Scw, ...),
// whose points compete for free slots, and orbfe_guided_best for Fuse and SearchBySim3, which keep each point's best
// candidate.  The map changes of the reference's accept loop are then replayed on the host in the original order.
// The cv::Mat algebra of the projections is written out element-wise with OpenCV 2.4's float/double semantics
// (a 3x3 * 3x1 gemm with flags 0 sums in float -- OpenCV's small-matrix path, pinned to cv2.gemm -- every other product
// in double; Mat/scalar scales by the float reciprocal).
// =================================================================================================
namespace ORB_SLAM {

namespace {

// A KeyFrame as the matchers' view.  KeyFrame keeps its image bounds and grid protected (KeyFrame.h:182-209), but they are
// Frame's: the constructor copies the bounds and grid cell sizes from Frame's statics (KeyFrame.cc:31-34), and mGrid is
// Frame's grid of mvKeysUn (:45-50), which the fused kernel rebuilds from the keys with the same bounds and cell sizes.  So
// the view takes them from Frame's statics, as make_view does, and a KeyFrame searched here must come from a Frame of the
// current image geometry.
struct KeyFrameView {
    KeyFrame *const pKF;
    const std::vector<cv::KeyPoint> keys;   // GetKeyPointsUn() and GetScaleFactors() return copies: they live here
    const std::vector<float> sf;
    const DescBuf desc;
    OrbfeFrameView v;
    explicit KeyFrameView(KeyFrame *kf) : pKF(kf), keys(kf->GetKeyPointsUn()), sf(kf->GetScaleFactors()), desc(kf->GetDescriptors()) {
        v.n = (int)keys.size();
        v.keys_un = v.n ? reinterpret_cast<const OrbfeKeyPoint *>(&keys[0]) : NULL;
        v.desc = desc.ptr;
        v.min_x = (float)Frame::mnMinX; v.min_y = (float)Frame::mnMinY;
        v.max_x = (float)Frame::mnMaxX; v.max_y = (float)Frame::mnMaxY;
        v.grid_inv_w = Frame::mfGridElementWidthInv;
        v.grid_inv_h = Frame::mfGridElementHeightInv;
        v.nlevels = pKF->GetScaleLevels();
        v.scale_factors = sf.empty() ? NULL : &sf[0];
    }
    // PredictScale: the first level whose factor is >= ratio, at most the last level
    int predict_level(float ratio) const { return std::min((int)(std::lower_bound(sf.begin(), sf.end(), ratio) - sf.begin()), v.nlevels - 1); }
};

template <typename T> const T *ptr_or_null(const std::vector<T> &v) { return v.empty() ? NULL : &v[0]; }

// the query windows of one call
struct Windows {
    std::vector<float> u, v, r;
    std::vector<int> lo, hi;
    std::vector<unsigned char> desc;
    int size() const { return (int)u.size(); }
    void add(float wu, float wv, float wr, int level, const cv::Mat &d) {
        u.push_back(wu); v.push_back(wv); r.push_back(wr);
        lo.push_back(level - 1); hi.push_back(level);
        desc.insert(desc.end(), d.ptr(0), d.ptr(0) + 32);
    }
    // orbfe_guided_best: best[q] = the feature query q keeps (best <= th_dist) or -1; false after a reported error
    bool best(const KeyFrameView &kf, int th_dist, std::vector<int> &best) const {
        best.assign(size() + 1, -1);
        return ok(orbfe_guided_best(thread_matcher(), &kf.v, size(), ptr_or_null(u), ptr_or_null(v), ptr_or_null(r), ptr_or_null(lo),
                                    ptr_or_null(hi), ptr_or_null(desc), th_dist, &best[0]));
    }
};

// y = R*x + t for 3x3 / 3x1 CV_32F Mats: one cv::gemm(R, x, 1, t, 1) with flags 0 -> OpenCV's unrolled small-matrix branch:
// the three products are summed in FLOAT, left to right, then (float)(sum + t) in double (pinned to cv2.gemm golden vectors,
// tests/golden/opencv_gemm.npz; this file is compiled with -ffp-contract=off)
void transform(const cv::Mat &R, const cv::Mat &t, const float x[3], float y[3])
{
    for (int k = 0; k < 3; k++) {
        float s = R.at<float>(k, 0) * x[0];
        s = s + R.at<float>(k, 1) * x[1];
        s = s + R.at<float>(k, 2) * x[2];
        y[k] = (float)((double)s + (double)t.at<float>(k, 0));
    }
}
void mat3(const cv::Mat &m, float out[3]) { for (int k = 0; k < 3; k++) out[k] = m.at<float>(k, 0); }
float norm3(const float v[3]) { return (float)std::sqrt((double)v[0] * v[0] + (double)v[1] * v[1] + (double)v[2] * v[2]); }

// Scw = [sR | st]: scw, Rcw = sRcw/scw, tcw = st/scw, Ow = -Rcw.t()*tcw   (ORBmatcher.cc:297-301, :1146-1150)
struct Sim3Cam {
    cv::Mat Rcw, tcw;
    float Ow[3];
    explicit Sim3Cam(const cv::Mat &Scw) {
        double dot = 0;
        for (int c = 0; c < 3; c++) dot += (double)Scw.at<float>(0, c) * (double)Scw.at<float>(0, c);
        const float scw = (float)std::sqrt(dot);
        const float inv = (float)(1.0 / (double)scw);  // Mat / scalar -> scale by 1./s
        Rcw.create(3, 3, CV_32F);
        tcw.create(3, 1, CV_32F);
        for (int r = 0; r < 3; r++) {
            for (int c = 0; c < 3; c++) Rcw.at<float>(r, c) = Scw.at<float>(r, c) * inv;
            tcw.at<float>(r, 0) = Scw.at<float>(r, 3) * inv;
        }
        for (int k = 0; k < 3; k++) {
            const double s = (double)Rcw.at<float>(0, k) * tcw.at<float>(0, 0) + (double)Rcw.at<float>(1, k) * tcw.at<float>(1, 0) +
                             (double)Rcw.at<float>(2, k) * tcw.at<float>(2, 0);
            Ow[k] = (float)(s * -1.0);
        }
    }
};

// shared gate of SearchByProjection(KF,Scw,..) and both Fuse overloads: returns false if the point is rejected; otherwise
// appends its query window
bool project(const KeyFrameView &kf, MapPoint *pMP, const cv::Mat &Rcw, const cv::Mat &tcw, const float Ow[3], float th,
             bool invz_in_double, Windows &w)
{
    KeyFrame *pKF = kf.pKF;
    float X[3], Xc[3];
    mat3(pMP->GetWorldPos(), X);
    transform(Rcw, tcw, X, Xc);
    if (Xc[2] < 0.0f) return false;  // depth must be positive
    const float invz = invz_in_double ? (float)(1.0 / (double)Xc[2]) : 1.0f / Xc[2];
    const float u = pKF->fx * (Xc[0] * invz) + pKF->cx;
    const float v = pKF->fy * (Xc[1] * invz) + pKF->cy;
    if (!pKF->IsInImage(u, v)) return false;
    const float maxDistance = pMP->GetMaxDistanceInvariance(), minDistance = pMP->GetMinDistanceInvariance();
    const float PO[3] = {X[0] - Ow[0], X[1] - Ow[1], X[2] - Ow[2]};
    const float dist = norm3(PO);
    if (dist < minDistance || dist > maxDistance) return false;
    float Pn[3];
    mat3(pMP->GetNormal(), Pn);
    const double dotPn = (double)PO[0] * Pn[0] + (double)PO[1] * Pn[1] + (double)PO[2] * Pn[2];  // Mat::dot: double
    if (dotPn < 0.5 * dist) return false;  // viewing angle < 60 deg
    const int nPredictedLevel = kf.predict_level(dist / minDistance);
    w.add(u, v, th * kf.sf[nPredictedLevel], nPredictedLevel, pMP->GetDescriptor());
    return true;
}

void feature_vector_csr(const DBoW2::FeatureVector &fv, std::vector<int> &ids, std::vector<int> &ptr, std::vector<int> &items)
{
    ids.clear(); ptr.assign(1, 0); items.clear();
    for (DBoW2::FeatureVector::const_iterator it = fv.begin(); it != fv.end(); ++it) {
        ids.push_back((int)it->first);
        for (size_t k = 0; k < it->second.size(); k++) items.push_back((int)it->second[k]);
        ptr.push_back((int)items.size());
    }
}

}  // namespace

// ---- Tracking::Relocalisation refinement (Tracking.cc:960,974) ------------------------------------------------
int ORBmatcher::SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, const std::set<MapPoint *> &sAlreadyFound, float th, int ORBdist)
{
    const DescBuf dc(CurrentFrame.mDescriptors);
    const OrbfeFrameView cur = make_view(CurrentFrame, dc);
    const std::vector<MapPoint *> vpMPs = pKF->GetMapPointMatches();
    const int np = (int)vpMPs.size();
    std::vector<unsigned char> valid(np + 1, 0), desc((size_t)np * 32 + 1, 0);
    std::vector<float> world((size_t)np * 3 + 1, 0.f), mind(np + 1, 1.f), ang(np + 1, 0.f);
    for (int i = 0; i < np; i++) {
        MapPoint *pMP = vpMPs[i];
        if (!pMP || pMP->isBad() || sAlreadyFound.count(pMP)) continue;  // :1642-1644
        valid[i] = 1;
        mat3(pMP->GetWorldPos(), &world[(size_t)i * 3]);
        mind[i] = pMP->GetMinDistanceInvariance();
        std::memcpy(&desc[(size_t)i * 32], pMP->GetDescriptor().ptr(0), 32);
        ang[i] = pKF->GetKeyPointUn(i).angle;
    }
    float T[12];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) T[4 * r + c] = CurrentFrame.mTcw.at<float>(r, c);
    std::vector<int> mp(cur.n > 0 ? cur.n : 1, -1);
    for (int i = 0; i < cur.n; i++)
        if (CurrentFrame.mvpMapPoints[i]) mp[i] = INT_MAX;
    int nmatches = 0;
    if (!ok(orbfe_search_by_projection_kf(thread_matcher(), &cur, np, &valid[0], &world[0], &mind[0], &desc[0], &ang[0], T, Frame::fx,
                                        Frame::fy, Frame::cx, Frame::cy, th, ORBdist, mbCheckOrientation ? 1 : 0, &mp[0], &nmatches))) return 0;
    for (int i = 0; i < cur.n; i++)
        if (mp[i] >= 0 && mp[i] != INT_MAX) CurrentFrame.mvpMapPoints[i] = vpMPs[mp[i]];
    return nmatches;
}

// ---- LoopClosing::ComputeSim3 (LoopClosing.cc:370) ------------------------------------------------------------
int ORBmatcher::SearchByProjection(KeyFrame *pKF, cv::Mat Scw, const std::vector<MapPoint *> &vpPoints, std::vector<MapPoint *> &vpMatched, int th)
{
    const KeyFrameView kf(pKF);
    const Sim3Cam cam(Scw);
    std::set<MapPoint *> spAlreadyFound(vpMatched.begin(), vpMatched.end());
    spAlreadyFound.erase(static_cast<MapPoint *>(NULL));
    Windows w;
    std::vector<int> q2mp;
    for (int iMP = 0, iend = (int)vpPoints.size(); iMP < iend; iMP++) {
        MapPoint *pMP = vpPoints[iMP];
        if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
        if (project(kf, pMP, cam.Rcw, cam.tcw, cam.Ow, (float)th, false, w)) q2mp.push_back(iMP);
    }
    // :373-398: the best candidate whose vpMatched entry is still empty (set on entry or by an earlier point), if <= TH_LOW
    std::vector<int> slot(kf.v.n + 1, -1);
    for (int i = 0; i < kf.v.n; i++)
        if (vpMatched[i]) slot[i] = INT_MAX;
    int nmatches = 0;
    if (!ok(orbfe_guided_search(thread_matcher(), &kf.v, w.size(), ptr_or_null(w.u), ptr_or_null(w.v), ptr_or_null(w.r),
                                ptr_or_null(w.lo), ptr_or_null(w.hi), ptr_or_null(w.desc), NULL, 0, 0.f, TH_LOW, 0, &slot[0],
                                &nmatches))) return 0;
    for (int i = 0; i < kf.v.n; i++)
        if (slot[i] >= 0 && slot[i] != INT_MAX) vpMatched[i] = vpPoints[q2mp[slot[i]]];
    return nmatches;
}

// ---- LocalMapping::SearchInNeighbors (LocalMapping.cc:405,430) --------------------------------------------------
int ORBmatcher::Fuse(KeyFrame *pKF, std::vector<MapPoint *> &vpMapPoints, float th)
{
    const cv::Mat Rcw = pKF->GetRotation(), tcw = pKF->GetTranslation();
    const KeyFrameView kf(pKF);
    float Ow[3];
    mat3(pKF->GetCameraCenter(), Ow);
    Windows w;
    std::vector<int> q2mp;
    for (size_t i = 0; i < vpMapPoints.size(); i++) {
        MapPoint *pMP = vpMapPoints[i];
        if (!pMP) continue;
        if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
        if (project(kf, pMP, Rcw, tcw, Ow, th, false, w)) q2mp.push_back((int)i);
    }
    std::vector<int> best;
    if (!w.best(kf, TH_LOW, best)) return 0;
    int nFused = 0;
    for (int q = 0; q < w.size(); q++) {  // :1090-1131
        const int bestIdx = best[q];
        if (bestIdx < 0) continue;
        MapPoint *pMP = vpMapPoints[q2mp[q]];
        // the reference evaluates this gate at the point's turn (:1040): a pointer listed twice is fused once
        if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
        MapPoint *pMPinKF = pKF->GetMapPoint(bestIdx);
        if (pMPinKF) { if (!pMPinKF->isBad()) pMP->Replace(pMPinKF); }
        else { pMP->AddObservation(pKF, bestIdx); pKF->AddMapPoint(pMP, bestIdx); }
        nFused++;
    }
    return nFused;
}

// ---- LoopClosing::SearchAndFuse (LoopClosing.cc:568) -------------------------------------------------------------
int ORBmatcher::Fuse(KeyFrame *pKF, cv::Mat Scw, const std::vector<MapPoint *> &vpPoints, float th)
{
    const KeyFrameView kf(pKF);
    const Sim3Cam cam(Scw);
    const std::set<MapPoint *> spAlreadyFound = pKF->GetMapPoints();
    Windows w;
    std::vector<int> q2mp;
    for (size_t iMP = 0; iMP < vpPoints.size(); iMP++) {
        MapPoint *pMP = vpPoints[iMP];
        if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
        if (project(kf, pMP, cam.Rcw, cam.tcw, cam.Ow, th, true, w)) q2mp.push_back((int)iMP);
    }
    std::vector<int> best;
    if (!w.best(kf, TH_LOW, best)) return 0;
    int nFused = 0;
    for (int q = 0; q < w.size(); q++) {  // :1222-1261
        const int bestIdx = best[q];
        if (bestIdx < 0) continue;
        MapPoint *pMP = vpPoints[q2mp[q]];
        MapPoint *pMPinKF = pKF->GetMapPoint(bestIdx);
        if (pMPinKF) { if (!pMPinKF->isBad()) pMPinKF->Replace(pMP); }
        else { pMP->AddObservation(pKF, bestIdx); pKF->AddMapPoint(pMP, bestIdx); }
        nFused++;
    }
    return nFused;
}

// ---- Tracking::Relocalisation / LoopClosing::ComputeSim3 (Tracking.cc:887, LoopClosing.cc:259) --------------------
int ORBmatcher::SearchByBoW(KeyFrame *pKF, Frame &F, std::vector<MapPoint *> &vpMapPointMatches)
{
    const std::vector<MapPoint *> vpMapPointsKF = pKF->GetMapPointMatches();
    vpMapPointMatches = std::vector<MapPoint *>(F.mvpMapPoints.size(), static_cast<MapPoint *>(NULL));
    std::vector<int> ids1, ptr1, it1, ids2, ptr2, it2;
    feature_vector_csr(pKF->GetFeatureVector(), ids1, ptr1, it1);
    feature_vector_csr(F.mFeatVec, ids2, ptr2, it2);
    const std::vector<cv::KeyPoint> k1 = pKF->GetKeyPointsUn();
    const int n1 = (int)vpMapPointsKF.size(), n2 = (int)F.mvKeys.size();
    std::vector<unsigned char> valid1(n1 + 1, 0), valid2(n2 + 1, 1);
    std::vector<float> a1(n1 + 1, 0.f), a2(n2 + 1, 0.f);
    for (int i = 0; i < n1; i++) { valid1[i] = vpMapPointsKF[i] && !vpMapPointsKF[i]->isBad(); a1[i] = k1[i].angle; }
    for (int i = 0; i < n2; i++) a2[i] = F.mvKeys[i].angle;  // :233 uses F.mvKeys
    const DescBuf d1(pKF->GetDescriptors()), d2(F.mDescriptors);
    std::vector<int> out(n2 + 1, -1);
    int nmatches = 0;
    if (!ok(orbfe_search_by_bow(thread_matcher(), 0, n1, d1.ptr, &valid1[0], &a1[0], (int)ids1.size(), ptr_or_null(ids1), &ptr1[0], ptr_or_null(it1),
                              n2, d2.ptr, &valid2[0], &a2[0], (int)ids2.size(), ptr_or_null(ids2), &ptr2[0], ptr_or_null(it2), mfNNratio,
                              mbCheckOrientation ? 1 : 0, &out[0], &nmatches))) return 0;
    for (int i2 = 0; i2 < n2; i2++)
        if (out[i2] >= 0) vpMapPointMatches[i2] = vpMapPointsKF[out[i2]];
    return nmatches;
}

int ORBmatcher::SearchByBoW(KeyFrame *pKF1, KeyFrame *pKF2, std::vector<MapPoint *> &vpMatches12)
{
    const std::vector<MapPoint *> vp1 = pKF1->GetMapPointMatches(), vp2 = pKF2->GetMapPointMatches();
    const std::vector<cv::KeyPoint> k1 = pKF1->GetKeyPointsUn(), k2 = pKF2->GetKeyPointsUn();
    vpMatches12 = std::vector<MapPoint *>(vp1.size(), static_cast<MapPoint *>(NULL));
    std::vector<int> ids1, ptr1, it1, ids2, ptr2, it2;
    feature_vector_csr(pKF1->GetFeatureVector(), ids1, ptr1, it1);
    feature_vector_csr(pKF2->GetFeatureVector(), ids2, ptr2, it2);
    const int n1 = (int)vp1.size(), n2 = (int)vp2.size();
    std::vector<unsigned char> valid1(n1 + 1, 0), valid2(n2 + 1, 0);
    std::vector<float> a1(n1 + 1, 0.f), a2(n2 + 1, 0.f);
    for (int i = 0; i < n1; i++) { valid1[i] = vp1[i] && !vp1[i]->isBad(); a1[i] = k1[i].angle; }
    for (int i = 0; i < n2; i++) { valid2[i] = vp2[i] && !vp2[i]->isBad(); a2[i] = k2[i].angle; }
    const DescBuf d1(pKF1->GetDescriptors()), d2(pKF2->GetDescriptors());
    std::vector<int> out(n1 + 1, -1);
    int nmatches = 0;
    if (!ok(orbfe_search_by_bow(thread_matcher(), 1, n1, d1.ptr, &valid1[0], &a1[0], (int)ids1.size(), ptr_or_null(ids1), &ptr1[0], ptr_or_null(it1),
                              n2, d2.ptr, &valid2[0], &a2[0], (int)ids2.size(), ptr_or_null(ids2), &ptr2[0], ptr_or_null(it2), mfNNratio,
                              mbCheckOrientation ? 1 : 0, &out[0], &nmatches))) return 0;
    for (int i1 = 0; i1 < n1; i1++)
        if (out[i1] >= 0) vpMatches12[i1] = vp2[out[i1]];
    return nmatches;
}

// ---- LocalMapping::CreateNewMapPoints (LocalMapping.cc:252) --------------------------------------------------------
bool ORBmatcher::CheckDistEpipolarLine(const cv::KeyPoint &kp1, const cv::KeyPoint &kp2, const cv::Mat &F12, const KeyFrame *pKF2)
{
    const float a = kp1.pt.x * F12.at<float>(0, 0) + kp1.pt.y * F12.at<float>(1, 0) + F12.at<float>(2, 0);
    const float b = kp1.pt.x * F12.at<float>(0, 1) + kp1.pt.y * F12.at<float>(1, 1) + F12.at<float>(2, 1);
    const float c = kp1.pt.x * F12.at<float>(0, 2) + kp1.pt.y * F12.at<float>(1, 2) + F12.at<float>(2, 2);
    const float num = a * kp2.pt.x + b * kp2.pt.y + c;
    const float den = a * a + b * b;
    if (den == 0) return false;
    const float dsqr = num * num / den;
    return dsqr < 3.84 * pKF2->GetSigma2(kp2.octave);
}

int ORBmatcher::SearchForTriangulation(KeyFrame *pKF1, KeyFrame *pKF2, cv::Mat F12, std::vector<cv::KeyPoint> &vMatchedKeys1,
                                       std::vector<cv::KeyPoint> &vMatchedKeys2, std::vector<std::pair<size_t, size_t> > &vMatchedPairs)
{
    const std::vector<MapPoint *> vp1 = pKF1->GetMapPointMatches(), vp2 = pKF2->GetMapPointMatches();
    const std::vector<cv::KeyPoint> k1 = pKF1->GetKeyPointsUn(), k2 = pKF2->GetKeyPointsUn();
    std::vector<int> ids1, ptr1, it1, ids2, ptr2, it2;
    feature_vector_csr(pKF1->GetFeatureVector(), ids1, ptr1, it1);
    feature_vector_csr(pKF2->GetFeatureVector(), ids2, ptr2, it2);
    const int n1 = (int)k1.size(), n2 = (int)k2.size();
    std::vector<unsigned char> has1(n1 + 1, 0), has2(n2 + 1, 0);
    for (int i = 0; i < n1; i++) has1[i] = vp1[i] != NULL;
    for (int i = 0; i < n2; i++) has2[i] = vp2[i] != NULL;
    float F[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) F[3 * r + c] = F12.at<float>(r, c);
    std::vector<float> sigma2(pKF2->GetScaleLevels());
    for (size_t l = 0; l < sigma2.size(); l++) sigma2[l] = pKF2->GetSigma2((int)l);
    const DescBuf d1(pKF1->GetDescriptors()), d2(pKF2->GetDescriptors());
    std::vector<int> m12(n1 + 1, -1);
    int nmatches = 0;
    if (!ok(orbfe_search_for_triangulation(thread_matcher(), n1, n1 ? reinterpret_cast<const OrbfeKeyPoint *>(&k1[0]) : NULL, d1.ptr, &has1[0],
                                         (int)ids1.size(), ptr_or_null(ids1), &ptr1[0], ptr_or_null(it1), n2,
                                         n2 ? reinterpret_cast<const OrbfeKeyPoint *>(&k2[0]) : NULL, d2.ptr, &has2[0], (int)ids2.size(),
                                         ptr_or_null(ids2), &ptr2[0], ptr_or_null(it2), F, &sigma2[0], mbCheckOrientation ? 1 : 0, &m12[0],
                                         &nmatches))) return 0;
    vMatchedKeys1.clear(); vMatchedKeys2.clear(); vMatchedPairs.clear();  // :994-1011
    for (int i = 0; i < n1; i++) {
        if (m12[i] < 0) continue;
        vMatchedKeys1.push_back(k1[i]);
        vMatchedKeys2.push_back(k2[m12[i]]);
        vMatchedPairs.push_back(std::make_pair((size_t)i, (size_t)m12[i]));
    }
    return nmatches;
}

// ---- LoopClosing::ComputeSim3 (LoopClosing.cc:317) ------------------------------------------------------------------
int ORBmatcher::SearchBySim3(KeyFrame *pKF1, KeyFrame *pKF2, std::vector<MapPoint *> &vpMatches12, const float &s12, const cv::Mat &R12,
                             const cv::Mat &t12, float th)
{
    const cv::Mat R1w = pKF1->GetRotation(), t1w = pKF1->GetTranslation(), R2w = pKF2->GetRotation(), t2w = pKF2->GetTranslation();
    // sR12 = s12*R12 ; sR21 = (1.0/s12)*R12.t() ; t21 = -sR21*t12   (:1282-1284)
    cv::Mat sR12(3, 3, CV_32F), sR21(3, 3, CV_32F), t21(3, 1, CV_32F);
    const float inv_s = (float)(1.0 / (double)s12);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) { sR12.at<float>(r, c) = R12.at<float>(r, c) * s12; sR21.at<float>(r, c) = R12.at<float>(c, r) * inv_s; }
    for (int k = 0; k < 3; k++) {   // -sR21*t12: gemm(sR21, t12, -1) with flags 0 -> the float small-matrix path, then * alpha
        float s = sR21.at<float>(k, 0) * t12.at<float>(0, 0);
        s = s + sR21.at<float>(k, 1) * t12.at<float>(1, 0);
        s = s + sR21.at<float>(k, 2) * t12.at<float>(2, 0);
        t21.at<float>(k, 0) = (float)((double)s * -1.0);
    }
    const std::vector<MapPoint *> vp1 = pKF1->GetMapPointMatches(), vp2 = pKF2->GetMapPointMatches();
    const int N1 = (int)vp1.size(), N2 = (int)vp2.size();
    std::vector<bool> done1(N1, false), done2(N2, false);
    for (int i = 0; i < N1; i++) {
        MapPoint *pMP = vpMatches12[i];
        if (!pMP) continue;
        done1[i] = true;
        const int idx2 = pMP->GetIndexInKeyFrame(pKF2);
        if (idx2 >= 0 && idx2 < N2) done2[idx2] = true;
    }
    std::vector<int> vnMatch1(N1, -1), vnMatch2(N2, -1);
    // one direction: project the points of `from` into `to` and take the best candidate (<= TH_HIGH)
    struct Dir { KeyFrame *from, *to; const cv::Mat *Rw, *tw, *sR, *t; const std::vector<MapPoint *> *vp; std::vector<bool> *done; std::vector<int> *match; };
    Dir dirs[2] = {{pKF1, pKF2, &R1w, &t1w, &sR21, &t21, &vp1, &done1, &vnMatch1}, {pKF2, pKF1, &R2w, &t2w, &sR12, &t12, &vp2, &done2, &vnMatch2}};
    for (int dsel = 0; dsel < 2; dsel++) {
        Dir &D = dirs[dsel];
        const KeyFrameView kf(D.to);
        Windows w;
        std::vector<int> q2i;
        for (int i = 0; i < (int)D.vp->size(); i++) {
            MapPoint *pMP = (*D.vp)[i];
            if (!pMP || (*D.done)[i]) continue;
            if (pMP->isBad()) continue;
            float X[3], Xa[3], Xb[3];
            mat3(pMP->GetWorldPos(), X);
            transform(*D.Rw, *D.tw, X, Xa);
            transform(*D.sR, *D.t, Xa, Xb);
            if (Xb[2] < 0.0f) continue;
            const float invz = (float)(1.0 / (double)Xb[2]);
            const float u = pKF1->fx * (Xb[0] * invz) + pKF1->cx, v = pKF1->fy * (Xb[1] * invz) + pKF1->cy;  // :1270-1273: KF1's intrinsics both ways
            if (!D.to->IsInImage(u, v)) continue;
            const float maxD = pMP->GetMaxDistanceInvariance(), minD = pMP->GetMinDistanceInvariance();
            const float dist3D = norm3(Xb);
            if (dist3D < minD || dist3D > maxD) continue;
            const int lv = kf.predict_level(dist3D / minD);
            w.add(u, v, th * kf.sf[lv], lv, pMP->GetDescriptor());
            q2i.push_back(i);
        }
        std::vector<int> best;
        if (!w.best(kf, TH_HIGH, best)) return 0;
        for (int q = 0; q < w.size(); q++)
            if (best[q] >= 0) (*D.match)[q2i[q]] = best[q];
    }
    int nFound = 0;  // :1486-1502: keep mutual agreements
    for (int i1 = 0; i1 < N1; i1++) {
        const int idx2 = vnMatch1[i1];
        if (idx2 >= 0 && vnMatch2[idx2] == i1) { vpMatches12[i1] = vp2[idx2]; nFound++; }
    }
    return nFound;
}

}  // namespace ORB_SLAM
