// oracle/ref_shim_slam: stand-in for the ROS image message the reference's Tracking.h names (never used by the drivers)
#ifndef ORB_REF_SHIM_SLAM_SENSOR_MSGS_IMAGE_H
#define ORB_REF_SHIM_SLAM_SENSOR_MSGS_IMAGE_H
namespace sensor_msgs {
struct Image {};
typedef const Image *ImageConstPtr;
}  // namespace sensor_msgs
#endif
