// oracle/ref_shim_lm: oracle/ref_shim/ros/ros.h plus the names LocalMapping.cc, FramePublisher.h and MapPublisher.h declare
// (LocalMapping::Run's rate loop, publisher members); the culling driver never runs them
#ifndef ORB_REF_SHIM_LM_ROS_H
#define ORB_REF_SHIM_LM_ROS_H
#include_next <ros/ros.h>
namespace ros {
struct Rate {
    explicit Rate(double) {}
    void sleep() {}
};
inline bool ok() { return false; }
struct NodeHandle {};
struct Publisher {};
}  // namespace ros
#endif
