// oracle/ref_shim_slam: stand-in for the ROS image encodings header (nothing of it is used by the drivers)
#ifndef ORB_REF_SHIM_SLAM_IMAGE_ENCODINGS_H
#define ORB_REF_SHIM_SLAM_IMAGE_ENCODINGS_H
namespace sensor_msgs {
namespace image_encodings {}
}  // namespace sensor_msgs
#endif
