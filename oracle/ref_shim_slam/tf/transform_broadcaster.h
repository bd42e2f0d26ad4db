// oracle/ref_shim_slam: stand-in for the tf broadcaster Tracking.h holds as a member.  Tracking's constructor publishes an
// identity transform through it, so these do nothing rather than abort; nothing is published.
#ifndef ORB_REF_SHIM_SLAM_TF_H
#define ORB_REF_SHIM_SLAM_TF_H
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
