// oracle/ref_shim_lm: stand-in for the ROS image encodings header (nothing of it is used on the culling path)
#ifndef ORB_REF_SHIM_LM_IMAGE_ENCODINGS_H
#define ORB_REF_SHIM_LM_IMAGE_ENCODINGS_H
namespace sensor_msgs {
namespace image_encodings {}
}  // namespace sensor_msgs
#endif
