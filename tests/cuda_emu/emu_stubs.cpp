// TEST INFRASTRUCTURE (emulated library only): level_tma_kernels.cu builds TMA tensor maps, which the CUDA-on-CPU shim does not
// model; without tensor maps the library uses resize_level_kernel + blur_level_kernel.
#include "rgbl_kernels.h"

namespace rgbl {
int make_level_tensor_maps(uint8_t*, size_t, int, const LevelGeom*, int, LevelTensorMaps* out) { out->n_levels = 0; return -1; }
int launch_level_tiles(cudaStream_t, const LevelTensorMaps&, uint8_t*, uint8_t*, size_t, const LevelGeom*, int, const LinCoef*, int) { return -1; }
}  // namespace rgbl
