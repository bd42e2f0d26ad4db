// oracle/ref_shim_lm/ref_lm_prelude.h -- force-included (-include) ahead of the reference's src/LocalMapping.cc when
// oracle/kf_culling.py compiles it for the culling driver (TEST INFRASTRUCTURE ONLY).  The OpenCV subset of
// oracle/ref_shim/ lacks what CreateNewMapPoints, ComputeF12 and SkewSymmetricMatrix use: cv::SVD, Mat::inv and the Mat_
// comma initialiser.  They are declared here with bodies that abort: the driver runs KeyFrameCulling only.  Mat::inv cannot
// be added to the shim's class from outside, so its one call (ComputeF12's return) is rewritten by a macro into a comma
// expression whose last operand aborts; the macro exists only in this translation unit.
#ifndef ORB_REF_SHIM_LM_PRELUDE_H
#define ORB_REF_SHIM_LM_PRELUDE_H
#include <cstdio>
#include <cstdlib>
#include <opencv2/core/core.hpp>

namespace cv {
inline Mat ref_lm_unreachable() {
    std::fprintf(stderr, "ref_kf_culling: a LocalMapping method other than KeyFrameCulling was called\n");
    std::abort();
}
struct SVD {
    enum { MODIFY_A = 1, NO_UV = 2, FULL_UV = 4 };
    static void compute(const Mat &, Mat &, Mat &, Mat &, int = 0) { ref_lm_unreachable(); }
};
struct RefLmCommaInit {
    template <class T>
    RefLmCommaInit operator,(const T &) const { return *this; }
    operator Mat() const { return ref_lm_unreachable(); }
};
template <class M, class T>
RefLmCommaInit operator<<(const Mat_<M> &, const T &) {
    ref_lm_unreachable();
    return RefLmCommaInit();
}
}  // namespace cv

#define inv() t(), ::cv::ref_lm_unreachable()
#endif
