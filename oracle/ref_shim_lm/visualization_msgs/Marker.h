// oracle/ref_shim_lm: stand-in for the marker message MapPublisher.h holds as members (never used on the culling path)
#ifndef ORB_REF_SHIM_LM_MARKER_H
#define ORB_REF_SHIM_LM_MARKER_H
namespace visualization_msgs {
struct Marker {};
}  // namespace visualization_msgs
#endif
