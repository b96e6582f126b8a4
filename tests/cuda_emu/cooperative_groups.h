// TEST INFRASTRUCTURE: the part of cooperative_groups the library's cluster kernel uses, over the CUDA-on-CPU shim (cuda_runtime.h).
#pragma once
#include "cuda_runtime.h"

namespace cooperative_groups {
struct cluster_group {
    unsigned block_rank() const { return emu::t_rank; }
    unsigned num_blocks() const { return emu::t_cluster->size; }
    void sync() const { emu::cluster_sync(); }
};
inline cluster_group this_cluster() { return {}; }
}  // namespace cooperative_groups
