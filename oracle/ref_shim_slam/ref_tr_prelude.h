// oracle/ref_shim_slam/ref_tr_prelude.h -- force-included (-include) by oracle/Makefile, after ref_lm_prelude.h, ahead of
// the reference's src/Tracking.cc for the local-map driver (TEST INFRASTRUCTURE ONLY).  The driver runs Tracking's
// constructor and UpdateReference() only; what the rest of Tracking.cc needs beyond the stand-ins of oracle/ref_shim/ and
// oracle/ref_shim_slam/ is declared here, and every body that a call other than those two could reach aborts.  Two names
// are rewritten by function-like macros that exist only in this translation unit (never in LocalMapping.cc's):
//   fSettings(path, mode)  the constructor's cv::FileStorage becomes a fixed settings table (the shim's FileStorage reads
//                          nothing and would give the ORBextractor zero levels)
//   worldPos(p)            CreateInitialMap's cv::Mat(Point3f), which the OpenCV stand-in lacks, aborts
#ifndef ORB_REF_SHIM_SLAM_TR_PRELUDE_H
#define ORB_REF_SHIM_SLAM_TR_PRELUDE_H
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <opencv2/core/core.hpp>

typedef struct RefTrCvMat CvMat;   // PnPsolver.h's private members name the OpenCV 1 C matrix
#define CV_RGB2GRAY 7
#define CV_BGR2GRAY 6

namespace ref_tr {
[[noreturn]] inline void unreachable(const char *what) {
    std::fprintf(stderr, "ref_local_map: %s is not linked\n", what);
    std::abort();
}

// the settings file the constructor reads: a pinhole camera without distortion and the extractor of the reference's
// example settings (1000 features, 8 levels at 1.2, FAST threshold 20, FAST score)
struct SettingsNode {
    double v;
    operator int() const { return (int)v; }
    operator float() const { return (float)v; }
    operator double() const { return v; }
};
struct Settings {
    SettingsNode operator[](const char *name) const {
        static const struct { const char *name; double v; } table[] = {
            {"Camera.fx", 500.0}, {"Camera.fy", 500.0}, {"Camera.cx", 320.0}, {"Camera.cy", 240.0}, {"Camera.k1", 0.0},
            {"Camera.k2", 0.0}, {"Camera.p1", 0.0}, {"Camera.p2", 0.0}, {"Camera.fps", 30.0}, {"Camera.RGB", 1.0},
            {"ORBextractor.nFeatures", 1000.0}, {"ORBextractor.scaleFactor", 1.2}, {"ORBextractor.nLevels", 8.0},
            {"ORBextractor.fastTh", 20.0}, {"ORBextractor.nScoreType", 1.0}, {"UseMotionModel", 1.0}};
        for (size_t i = 0; i < sizeof(table) / sizeof(table[0]); i++)
            if (std::strcmp(table[i].name, name) == 0) return SettingsNode{table[i].v};
        std::fprintf(stderr, "ref_local_map: no setting %s\n", name);
        std::abort();
    }
};

inline cv::Mat point_mat(const cv::Point3f &) { unreachable("cv::Mat(cv::Point3f)"); }
}  // namespace ref_tr

namespace cv {
template <class A, class B>
void cvtColor(const A &, B &, int) { ::ref_tr::unreachable("cv::cvtColor"); }
}  // namespace cv

#define fSettings(path, mode) fSettings_file(path, mode); const ::ref_tr::Settings fSettings
#define worldPos(p) worldPos = ::ref_tr::point_mat(p)
#endif
