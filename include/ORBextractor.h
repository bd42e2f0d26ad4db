/*
 * ORBextractor.h -- API-compatible replacement of ORB_SLAM's extractor header (raulmur/ORB_SLAM v1.0.1,
 * include/ORBextractor.h:32-77): same enum, constructor defaults, call operator and accessors, so that
 * Frame.cc:60,92-93 and Tracking.cc:111,126 compile against it unchanged.
 *
 * Implementation: orb_slam_b200/host/ORBextractor.cc forwards to the C-ABI of liborbfe.so (include/orbfe.h);
 * pyramid, FAST, retention, orientation, blur and rBRIEF run as hand-written sm_90a CUDA kernels.
 * No CPU fallback: constructing an extractor without a usable CUDA device terminates with a message.
 */
#ifndef ORBEXTRACTOR_H
#define ORBEXTRACTOR_H

#include <list>
#include <vector>

#include <opencv/cv.h>

struct OrbfeExtractor;  // opaque handle owned by liborbfe.so

namespace ORB_SLAM {

class ORBextractor {
public:
    enum { HARRIS_SCORE = 0, FAST_SCORE = 1 };

    ORBextractor(int nfeatures = 1000, float scaleFactor = 1.2f, int nlevels = 8, int scoreType = FAST_SCORE, int fastTh = 20);
    ~ORBextractor();

    // keypoints + 32-byte descriptors of one CV_8UC1 image.  `mask` has no effect, as in the reference: ORBextractor.cc:601-603
    // builds a cellMask that no call consumes (cv::FAST runs unmasked, :607), and Frame.cc:60 passes cv::Mat()
    void operator()(cv::InputArray image, cv::InputArray mask, std::vector<cv::KeyPoint>& keypoints, cv::OutputArray descriptors);

    int inline GetLevels() { return nlevels; }
    float inline GetScaleFactor() { return scaleFactor; }

    // CUDA device used by extractors constructed afterwards (default 0); extension, not in the reference
    static void SetDevice(int device);

    // What a failing liborbfe call does (extension, same contract as ORBmatcher::SetErrorHandler): the handler is called
    // with the OrbfeStatus code and message, then operator() returns no keypoints.  Default: log to stderr, abort only if
    // ORBFE_ABORT_ON_ERROR is set.  NULL restores the default.
    typedef void (*ErrorHandler)(int code, const char *message);
    static void SetErrorHandler(ErrorHandler handler);

protected:
    int nfeatures;
    double scaleFactor;  // a double initialised from the float argument, exactly like the reference member
    int nlevels;
    int scoreType;
    int fastTh;
    OrbfeExtractor* mpImpl;  // stands in for the reference's tables and scratch pyramids

private:
    ORBextractor(const ORBextractor&);             // the handle owns device memory: not copyable
    ORBextractor& operator=(const ORBextractor&);
};

}  // namespace ORB_SLAM

#endif  // ORBEXTRACTOR_H
