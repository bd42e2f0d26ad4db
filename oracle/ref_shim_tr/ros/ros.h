// oracle/ref_shim_tr: oracle/ref_shim_lm/ros/ros.h plus the names Tracking.cc takes from ROS: ros::Time for the
// constructor's transform (a no-op there), and the subscriber of Tracking::Run, which aborts if reached.  The NodeHandle of
// ref_shim_lm has no subscribe(), so it is renamed while that header is read and replaced by the one below.
#ifndef ORB_REF_SHIM_TR_ROS_H
#define ORB_REF_SHIM_TR_ROS_H
#define NodeHandle NodeHandleLm
#include_next <ros/ros.h>
#undef NodeHandle
namespace ros {
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
