// Host-side tensor-map encoding shared by the pyramid kernels and the matcher.
#pragma once
#include <cuda.h>          // CUtensorMap (types only: the encoder is fetched through the runtime, no libcuda link)
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace psb {

// 2-D float tensor of w x h elements, rows `pitch_bytes` apart, box of box_w x box_h elements; elements outside the
// tensor read as zero.  swizzle128: CU_TENSOR_MAP_SWIZZLE_128B (box_w * 4 must then be 128 bytes), else no swizzle.
// cuTensorMapEncodeTiled is a host-side encoder: it is fetched with cudaGetDriverEntryPoint, so the library does not
// link against libcuda.  Returns false when the driver does not offer it or rejects the arguments.
bool make_tmap_2d(CUtensorMap* map, const float* base, int w, int h, size_t pitch_bytes, int box_w, int box_h, bool swizzle128);
// the same for a 2-D uint8 tensor (w x h bytes; with swizzle128, box_w must be 128)
bool make_tmap_2d(CUtensorMap* map, const uint8_t* base, int w, int h, size_t pitch_bytes, int box_w, int box_h, bool swizzle128);

} // namespace psb
