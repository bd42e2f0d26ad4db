// vocab.h -- the device node table behind OrbfeVocabulary, shared by its two constructors: orbfe_vocabulary_create
// (bow_kernels.cu, host arrays) and orbfe_vocabulary_load_text (vocab_text.cu, DBoW2 text parsed on the device).
// Not part of the public ABI.
#pragma once

#include <mutex>

#include "../../include/orbfe_bow.h"
#include "orbfe_internal.h"

struct OrbfeVocabulary {
    int device = 0, nnodes = 0, depth = 0, weighting = 0, norm = 0;
    int k = -1, scoring = -1;       // header fields of a loaded text; create() never receives them
    int nwords = 0;                 // largest word id + 1
    int nchild = 0;                 // entries of d_children (child_ptr[nnodes])
    cudaStream_t stream = nullptr;
    orbfe::DeviceBuffers mem;       // the node table below
    uint8_t *d_desc = nullptr;
    uint8_t *d_live = nullptr;      // per node: weight > 0 (the FeatureVector skips stopped words)
    int *d_child_ptr = nullptr, *d_children = nullptr;
    int *d_word_id = nullptr;       // per node, for the BowVector kernel
    double *d_weight = nullptr;
    // the host-array entries stage through `stage` on `stream`, one call at a time
    std::mutex mu;
    orbfe::Stage stage;
};

namespace orbfe {
// Creates the vocabulary's stream and allocates its node table for `nnodes` nodes and `nchild` child entries on v->device
// (already current).  On failure the caller hands v to orbfe_vocabulary_destroy, which frees whatever was allocated.
cudaError_t vocab_alloc(OrbfeVocabulary *v, int nnodes, int nchild);
}  // namespace orbfe
