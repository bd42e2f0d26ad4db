// oracle/ref_shim_slam: stand-in for the marker message MapPublisher.h holds as members (never used by the drivers)
#ifndef ORB_REF_SHIM_SLAM_MARKER_H
#define ORB_REF_SHIM_SLAM_MARKER_H
namespace visualization_msgs {
struct Marker {};
}  // namespace visualization_msgs
#endif
