#include "tma_util.h"

namespace psb {

namespace {

bool encode_2d(CUtensorMap* map, CUtensorMapDataType type, const void* base, int w, int h, size_t pitch_bytes, int box_w, int box_h,
               bool swizzle128)
{
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static const EncodeFn encode = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            p = nullptr;
        }
        return reinterpret_cast<EncodeFn>(p);
    }();
    if (!encode) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)w, (cuuint64_t)h};
    const cuuint64_t strides[1] = {(cuuint64_t)pitch_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_h};
    const cuuint32_t estr[2] = {1, 1};
    return encode(map, type, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

} // namespace

bool make_tmap_2d(CUtensorMap* map, const float* base, int w, int h, size_t pitch_bytes, int box_w, int box_h, bool swizzle128)
{
    return encode_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, w, h, pitch_bytes, box_w, box_h, swizzle128);
}

bool make_tmap_2d(CUtensorMap* map, const uint8_t* base, int w, int h, size_t pitch_bytes, int box_w, int box_h, bool swizzle128)
{
    return encode_2d(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, w, h, pitch_bytes, box_w, box_h, swizzle128);
}

} // namespace psb
