// oracle/ref_shim/ref_voc_nodes.cc -- extern "C" driver of the reference's OWN TemplatedVocabulary::loadFromTextFile
// (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1338-1424), the call of src/main.cc (TEST INFRASTRUCTURE ONLY).
//
// Built by oracle/Makefile into oracle/_ref/libref_drivers.so, linked against libref_orbslam.so (the reference's DBoW2
// compiled unmodified).  m_nodes is protected: a class derived from ORBVocabulary reads it out, field for field.
#include <opencv2/core/core.hpp>

#include <chrono>
#include <cstring>

#include "ORBVocabulary.h"

using namespace ORB_SLAM;

namespace {
struct NodesVocabulary : public ORBVocabulary {
    using ORBVocabulary::m_nodes;
    using ORBVocabulary::m_k;
    using ORBVocabulary::m_L;
    using ORBVocabulary::m_scoring;
    using ORBVocabulary::m_weighting;
};
}  // namespace

extern "C" {

// NULL when loadFromTextFile returns false; *seconds (may be NULL) = its wall time
void *ref_voc_nodes_load(const char *path, double *seconds) {
    NodesVocabulary *v = new NodesVocabulary();
    const auto t0 = std::chrono::steady_clock::now();
    const bool ok = v->loadFromTextFile(path);
    if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (!ok) { delete v; return NULL; }
    return v;
}

void ref_voc_nodes_free(void *h) { delete static_cast<NodesVocabulary *>(h); }

// header fields, m_nodes.size(), the total number of children and m_words.size()
void ref_voc_nodes_info(void *h, int *k, int *L, int *scoring, int *weighting, int *nnodes, int *nchildren, int *nwords) {
    NodesVocabulary *v = static_cast<NodesVocabulary *>(h);
    *k = v->m_k;
    *L = v->m_L;
    *scoring = (int)v->m_scoring;
    *weighting = (int)v->m_weighting;
    *nnodes = (int)v->m_nodes.size();
    size_t nc = 0;
    for (const auto &n : v->m_nodes) nc += n.children.size();
    *nchildren = (int)nc;
    *nwords = (int)v->size();
}

// m_nodes as CSR: node i's children at children[child_ptr[i] .. child_ptr[i+1]) in m_nodes[i].children order; a node
// without a descriptor (the root) gets 32 zero bytes
void ref_voc_nodes_export(void *h, unsigned char *desc, int *child_ptr, int *children, int *word_id, double *weight, int *parent) {
    NodesVocabulary *v = static_cast<NodesVocabulary *>(h);
    int c = 0;
    for (size_t i = 0; i < v->m_nodes.size(); i++) {
        const auto &n = v->m_nodes[i];
        child_ptr[i] = c;
        for (unsigned ch : n.children) children[c++] = (int)ch;
        word_id[i] = (int)n.word_id;
        weight[i] = n.weight;
        parent[i] = (int)n.parent;
        if (n.descriptor.empty()) memset(desc + 32 * i, 0, 32);
        else memcpy(desc + 32 * i, n.descriptor.ptr<unsigned char>(), 32);
    }
    child_ptr[v->m_nodes.size()] = c;
}

}  // extern "C"
