// oracle/ref_shim_lm: stand-in for the tf broadcaster Tracking.h holds as a member (never used on the culling path)
#ifndef ORB_REF_SHIM_LM_TF_H
#define ORB_REF_SHIM_LM_TF_H
namespace tf {
struct TransformBroadcaster {};
}  // namespace tf
#endif
