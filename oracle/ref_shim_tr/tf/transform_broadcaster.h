// oracle/ref_shim_tr: stand-in for the tf broadcaster.  Tracking's constructor publishes an identity transform through it,
// so these do nothing rather than abort; nothing is published.
#ifndef ORB_REF_SHIM_TR_TF_H
#define ORB_REF_SHIM_TR_TF_H
#define ORB_REF_SHIM_LM_TF_H   // oracle/ref_shim_lm/tf/transform_broadcaster.h: this header replaces it
#include <ros/ros.h>
namespace tf {
struct Matrix3x3 {
    Matrix3x3(double, double, double, double, double, double, double, double, double) {}
};
struct Vector3 {
    Vector3(double, double, double) {}
};
struct Transform {
    Transform() {}
    Transform(const Matrix3x3 &, const Vector3 &) {}
    void setIdentity() {}
};
struct StampedTransform {
    StampedTransform(const Transform &, const ros::Time &, const char *, const char *) {}
};
struct TransformBroadcaster {
    void sendTransform(const StampedTransform &) {}
};
}  // namespace tf
#endif
