// oracle/ref_shim_lm: the two names LoopClosing.h and Optimizer.h take from g2o / Eigen (a map type and its members; no
// similarity transform is computed on the culling path)
#ifndef ORB_REF_SHIM_LM_G2O_SIM3_H
#define ORB_REF_SHIM_LM_G2O_SIM3_H
#include <memory>
namespace g2o {
class Sim3 {};
}  // namespace g2o
namespace Eigen {
template <class T>
class aligned_allocator : public std::allocator<T> {
public:
    template <class U>
    struct rebind {
        typedef aligned_allocator<U> other;
    };
    aligned_allocator() {}
    template <class U>
    aligned_allocator(const aligned_allocator<U> &) {}
};
}  // namespace Eigen
#endif
