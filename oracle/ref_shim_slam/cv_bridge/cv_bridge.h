// oracle/ref_shim_slam: stand-in for cv_bridge, which Tracking::GrabImage uses to read a ROS image (never reached by the
// local-map driver)
#ifndef ORB_REF_SHIM_SLAM_CV_BRIDGE_H
#define ORB_REF_SHIM_SLAM_CV_BRIDGE_H
#include <opencv2/core/core.hpp>
#include <sensor_msgs/Image.h>
namespace cv_bridge {
struct Exception {
    const char *what() const { return "cv_bridge stand-in"; }
};
struct Stamp {
    double toSec() const { return 0.0; }
};
struct Header {
    Stamp stamp;
};
struct CvImage {
    cv::Mat image;
    Header header;
};
typedef const CvImage *CvImageConstPtr;
inline CvImageConstPtr toCvShare(const sensor_msgs::ImageConstPtr &) {
    std::fprintf(stderr, "ref_local_map: cv_bridge::toCvShare is not linked\n");
    std::abort();
}
}  // namespace cv_bridge
#endif
