// oracle/ref_shim_slam: oracle/ref_shim/ros/ros.h plus the names the reference's thread classes take from ROS:
// LocalMapping::Run's rate loop, the publisher members of FramePublisher.h and MapPublisher.h, ros::Time for Tracking's
// constructor (a no-op there), and the subscriber and spin of Tracking::Run, which abort if reached.  The drivers never
// run Run.
#ifndef ORB_REF_SHIM_SLAM_ROS_H
#define ORB_REF_SHIM_SLAM_ROS_H
#include_next <ros/ros.h>
namespace ros {
struct Rate {
    explicit Rate(double) {}
    void sleep() {}
};
inline bool ok() { return false; }
struct Publisher {};
struct Time {
    static Time now() { return Time(); }
};
struct Subscriber {};
struct NodeHandle {
    template <class... A>
    Subscriber subscribe(A...) {
        std::fprintf(stderr, "ref_local_map: ros::NodeHandle::subscribe is not linked\n");
        std::abort();
    }
};
inline void spin() {
    std::fprintf(stderr, "ref_local_map: ros::spin is not linked\n");
    std::abort();
}
}  // namespace ros
#endif
