// The reference's alternative descriptor extraction modes (Config::DescMode, --desc-mode), for sm_90a:
//   grid    16 x 16 sample points per cell on the rotated grid, each rounded to the nearest pixel, point-sampled gradient
//           (reference src/popsift/s_desc_grid.cu:18-122)
//   igrid   the same grid, unrounded; gradient from four bilinearly interpolated samples one pixel along / across the
//           keypoint orientation; weights from the desc_gauss / desc_tile tables (s_desc_igrid.cu:18-72)
//   iloop   the `loop` scan over the cell's bounding box in 32 x 32 steps with the interpolated, rotated gradient
//           (s_desc_iloop.cu:18-124)
//   notile  igrid's samples, a different thread mapping and summation order (s_desc_notile.cu:26-87)
// They are sampling schemes, not hot paths: one CTA of 256 threads per descriptor (pulled from the device-side work
// counter like descriptor_kernel), thread <-> sample mapping, per-lane accumulation order and shuffle reductions as in
// the reference, so that descriptors agree to the last bits the texture arithmetic allows; normalisation is fused
// (k_desc_norm.h).  The reference reads the Gaussian planes through textures: point sampling = clamped integer
// addressing; linear sampling = the B200 float-texture blend measured with oracle/texprobe.cu (8-bit fractions and
// weights, tests/golden/texture_float.npz), evaluated here in float32 (descriptor tolerance 1e-3; the difference to the
// exactly rounded blend is < 1e-7 relative).
#include "ps_internal.h"
#include "k_desc_norm.h"

#include <cmath>
#include <mutex>

namespace psb {

namespace {

__constant__ float c_desc_gauss[40 * 40];     // reference sift_constants.cu:34-43
__constant__ float c_desc_tile[16];           // reference sift_constants.cu:45-48

__device__ const float kPi2d = 2.0f * 3.14159265358979323846f;
__device__ const float k4RPi = 4.0f / 3.14159265358979323846f;

struct Plane { const float* p; int w, h, pitch; };

// tex2DLayered point sampling at (x + 0.5, y + 0.5), clamp addressing (reference assist.h:69-77)
__device__ __forceinline__ float tex_point(const Plane& pl, int x, int y)
{
    x = min(max(x, 0), pl.w - 1);
    y = min(max(y, 0), pl.h - 1);
    return __ldg(pl.p + (size_t)y * pl.pitch + x);
}

// tex2DLayered linear sampling at (x + 0.5, y + 0.5): texel-space coordinate x, 8-bit fraction (round half up),
// 8-bit blend weights, clamp addressing
__device__ __forceinline__ float tex_linear(const Plane& pl, float x, float y)
{
    float fx = __fsub_rn(__fadd_rn(x, 0.5f), 0.5f), fy = __fsub_rn(__fadd_rn(y, 0.5f), 0.5f);
    fx = fminf(fmaxf(fx, -0.5f), (float)pl.w - 0.5f);
    fy = fminf(fmaxf(fy, -0.5f), (float)pl.h - 0.5f);
    const float flx = floorf(fx), fly = floorf(fy);
    int ix = (int)flx, iy = (int)fly;
    int ax = (int)floorf(__fmaf_rn(fx - flx, 256.0f, 0.5f)), ay = (int)floorf(__fmaf_rn(fy - fly, 256.0f, 0.5f));
    if (ax == 256) { ax = 0; ix += 1; }
    if (ay == 256) { ay = 0; iy += 1; }
    const int x0 = min(max(ix, 0), pl.w - 1), x1 = min(max(ix + 1, 0), pl.w - 1);
    const int y0 = min(max(iy, 0), pl.h - 1), y1 = min(max(iy + 1, 0), pl.h - 1);
    const float* r0 = pl.p + (size_t)y0 * pl.pitch;
    const float* r1 = pl.p + (size_t)y1 * pl.pitch;
    const int w11 = (ax * ay + 128) >> 8, w10 = ax - w11, w01 = ay - w11, w00 = 256 - ax - ay + w11;
    float s = __fmul_rn((float)w00, __ldg(r0 + x0));
    s = __fmaf_rn((float)w10, __ldg(r0 + x1), s);
    s = __fmaf_rn((float)w01, __ldg(r1 + x0), s);
    s = __fmaf_rn((float)w11, __ldg(r1 + x1), s);
    return __fmul_rn(s, 1.0f / 256.0f);
}

// reference s_gradiant.h:72-84 (point) and :86-104 (interpolated, along / across the keypoint orientation)
__device__ __forceinline__ void gradient_point(const Plane& pl, int x, int y, float& mod, float& th)
{
    const float dx = __fsub_rn(tex_point(pl, x + 1, y), tex_point(pl, x - 1, y));
    const float dy = __fsub_rn(tex_point(pl, x, y + 1), tex_point(pl, x, y - 1));
    mod = hypotf(dx, dy);
    th = atan2f(dy, dx);
}
__device__ __forceinline__ void gradient_rot(const Plane& pl, float x, float y, float cos_t, float sin_t, float& mod, float& th)
{
    const float dx = __fsub_rn(tex_linear(pl, x + cos_t, y + sin_t), tex_linear(pl, x - cos_t, y - sin_t));
    const float dy = __fsub_rn(tex_linear(pl, x - sin_t, y + cos_t), tex_linear(pl, x + sin_t, y - cos_t));
    mod = hypotf(dx, dy);
    th = atan2f(dy, dx);
}

constexpr int MT = 256;         // threads per descriptor

template <int MODE>
__global__ void __launch_bounds__(MT)
desc_mode_kernel(PyramidView pyr, Consts k, const ps_extremum* __restrict__ ext, const int* __restrict__ feat_to_ext,
                 ps_descriptor* __restrict__ desc, Counters* ct)
{
    __shared__ __align__(16) float raw[128];
    __shared__ int next_d;
    const int total = ct->ori_total;
    const int lane = threadIdx.x & 31;
    for (;;) {
        if (threadIdx.x == 0) next_d = atomicAdd(&ct->work_desc, 1);
        __syncthreads();
        const int d = next_d;
        if (d >= total) break;
        const int ei = feat_to_ext[d];
        const ps_extremum e = ext[ei];
        const float ang = e.orientation[min(max(d - e.idx_ori, 0), PS_MAX_ORI - 1)];
        const OctaveView& ov = pyr.oct[e.octave];
        Plane pl;
        pl.w = ov.w; pl.h = ov.h; pl.pitch = ov.pitch;
        pl.p = ov.gauss + (size_t)min(max(e.lpos, 0), pyr.levels + 2) * ov.plane;
        const float x = e.xpos, y = e.ypos;
        const float SBP = fabsf(3.0f * e.sigma);
        if (threadIdx.x < 128) raw[threadIdx.x] = 0.0f;
        __syncthreads();
        if (SBP != 0.0f) {
            float sin_t, cos_t;
            __sincosf(ang, &sin_t, &cos_t);
            if (MODE == PS_DESC_GRID) {
                // half-warp = cell (ix, iy); lane xd walks yd = 0..15 (s_desc_grid.cu:57-105)
                const int cell = threadIdx.x >> 4, xd = threadIdx.x & 15;
                const int ix = cell & 3, iy = cell >> 2;
                const float csbp = cos_t * SBP, ssbp = sin_t * SBP;
                const float offx = (float)ix - 1.5f, offy = (float)iy - 1.5f;
                const float ptx = fmaf(csbp, offx, fmaf(-ssbp, offy, x)), pty = fmaf(csbp, offy, fmaf(ssbp, offx, y));
                const float ldx = -cos_t + sin_t, ldy = -cos_t - sin_t;            // lft_dn
                const float rsx = cos_t / 8.0f, rsy = sin_t / 8.0f, usx = -sin_t / 8.0f, usy = cos_t / 8.0f;
                float dpt[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                for (int yd = 0; yd < 16; ++yd) {
                    float pox = ldx + ((float)xd + 0.5f) * rsx + ((float)yd + 0.5f) * usx;
                    float poy = ldy + ((float)xd + 0.5f) * rsy + ((float)yd + 0.5f) * usy;
                    float pixx = pox * SBP, pixy = poy * SBP;
                    pixx = roundf(ptx + pixx) - ptx;
                    pixy = roundf(pty + pixy) - pty;
                    pox = pixx / SBP; poy = pixy / SBP;
                    float mod, th;
                    gradient_point(pl, (int)(ptx + pixx), (int)(pty + pixy), mod, th);
                    const float nx = fmaf(cos_t, pox, sin_t * poy), ny = fmaf(cos_t, poy, -sin_t * pox);
                    const float dnx = nx + offx, dny = ny + offy;
                    const float ww = expf(-scalbnf(dnx * dnx + dny * dny, -3));
                    const float wx = 1.0f - fabsf(nx), wy = 1.0f - fabsf(ny);
                    if (wx < 0.0f || wy < 0.0f) continue;
                    const float wgt = ww * wx * wy * mod;
                    th -= ang;
                    th += (th < 0.0f ? kPi2d : 0.0f);
                    th -= (th >= kPi2d ? kPi2d : 0.0f);
                    const float tth = __fmul_ru(th, k4RPi);
                    const int fo0 = (int)floorf(tth);
                    const float do0 = tth - (float)fo0;
                    const int fo = fo0 % 8;
#pragma unroll
                    for (int b = 0; b < 8; ++b) {                                    // dpt[fo] / dpt[fo + 1] without dynamic indexing
                        if (fo == b) { dpt[b] = __fmaf_ru(1.0f - do0, wgt, dpt[b]); dpt[b + 1] = __fmaf_ru(do0, wgt, dpt[b + 1]); }
                    }
                }
                dpt[0] += dpt[8];
#pragma unroll
                for (int b = 0; b < 8; ++b) {
                    dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 8, 16);
                    dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 4, 16);
                    dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 2, 16);
                    dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 1, 16);
                }
                if (xd == 0)
#pragma unroll
                    for (int b = 0; b < 8; ++b) raw[cell * 8 + b] = dpt[b];
            } else if (MODE == PS_DESC_IGRID) {
                // half-warp = cell; lane xd walks yd = 0..15 (s_desc_igrid.cu:30-63)
                const int cell = threadIdx.x >> 4, xd = threadIdx.x & 15;
                const int ix = cell & 3, iy = cell >> 2;
                float dpt[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                for (int yd = 0; yd < 16; ++yd) {
                    const float stepx = (float)ix - 2.5f + 1.0f / 16.0f + (float)xd / 8.0f;
                    const float stepy = (float)iy - 2.5f + 1.0f / 16.0f + (float)yd / 8.0f;
                    const float ptx = cos_t * stepx + -sin_t * stepy;
                    const float pty = cos_t * stepy + sin_t * stepx;
                    float mod, th;
                    gradient_rot(pl, x + ptx * SBP, y + pty * SBP, cos_t, sin_t, mod, th);
                    th += (th < 0.0f ? kPi2d : 0.0f);
                    th -= (th >= kPi2d ? kPi2d : 0.0f);
                    const float ww = c_desc_gauss[(iy * 8 + yd) * 40 + ix * 8 + xd];
                    const float wgt = ww * c_desc_tile[xd] * c_desc_tile[yd] * mod;
                    const float tth = __fmul_ru(th, k4RPi);
                    const int fo = (int)floorf(tth);
                    const float do0 = tth - (float)fo;
                    const int fo1 = (fo + 1) & 7, fo0 = fo & 7;
#pragma unroll
                    for (int b = 0; b < 8; ++b) {
                        if (fo1 == b) dpt[b] = dpt[b] + wgt * do0;
                    }
#pragma unroll
                    for (int b = 0; b < 8; ++b) {
                        if (fo0 == b) dpt[b] = dpt[b] + wgt * (1.0f - do0);
                    }
                }
#pragma unroll
                for (int b = 0; b < 8; ++b) {
                    dpt[b] += __shfl_xor_sync(0xffffffffu, dpt[b], 1, 16);
                    dpt[b] += __shfl_xor_sync(0xffffffffu, dpt[b], 2, 16);
                    dpt[b] += __shfl_xor_sync(0xffffffffu, dpt[b], 4, 16);
                    dpt[b] += __shfl_xor_sync(0xffffffffu, dpt[b], 8, 16);
                }
                if (xd == 0)
#pragma unroll
                    for (int b = 0; b < 8; ++b) raw[cell * 8 + b] = dpt[b];
            } else if (MODE == PS_DESC_ILOOP) {
                // warp = cell, lane j walks i = 0..31; the 8 warps take two cells each (s_desc_iloop.cu:42-108)
                const float csbp = cos_t * SBP, ssbp = sin_t * SBP;
                const float bsz = fabsf(cos_t) + fabsf(sin_t);
                for (int cell = threadIdx.x >> 5; cell < 16; cell += MT / 32) {
                    const int ix = cell & 3, iy = cell >> 2;
                    const float offx = (float)ix - 1.5f, offy = (float)iy - 1.5f;
                    const float ptx = fmaf(csbp, offx, -ssbp * offy), pty = fmaf(csbp, offy, ssbp * offx);
                    float dpt[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                    const int j = lane;
                    for (int i = 0; i < 32; ++i) {
                        const float dx = -bsz + (float)j * bsz / 16.0f;
                        const float dy = -bsz + (float)i * bsz / 16.0f;
                        const float nx = fmaf(cos_t, dx, sin_t * dy), ny = fmaf(cos_t, dy, -sin_t * dx);
                        const float anx = fabsf(nx), any = fabsf(ny);
                        if (anx < 1.0f && any < 1.0f) {
                            const float jj = x + ptx + dx * SBP, ii = y + pty + dy * SBP;
                            float mod, th;
                            gradient_rot(pl, jj, ii, cos_t, sin_t, mod, th);
                            const float dnx = nx + offx, dny = ny + offy;
                            const float ww = __expf(-scalbnf(dnx * dnx + dny * dny, -3));
                            const float wgt = ww * (1.0f - anx) * (1.0f - any) * mod;
                            th += (th < 0.0f ? kPi2d : 0.0f);
                            th -= (th >= kPi2d ? kPi2d : 0.0f);
                            const float tth = __fmul_ru(th, k4RPi);
                            const int fo0 = (int)floorf(tth);
                            const float do0 = tth - (float)fo0;
                            const int fo = fo0 % 8;
#pragma unroll
                            for (int b = 0; b < 8; ++b) {
                                if (fo == b) { dpt[b] = __fmaf_ru(1.0f - do0, wgt, dpt[b]); dpt[b + 1] = __fmaf_ru(do0, wgt, dpt[b + 1]); }
                            }
                        }
                    }
                    dpt[0] += dpt[8];
#pragma unroll
                    for (int b = 0; b < 8; ++b) {
                        dpt[b] = tree_down(dpt[b]);
                        if (lane == 0) raw[cell * 8 + b] = dpt[b];
                    }
                }
            } else {   // PS_DESC_NOTILE
                // the reference's block is (32, 4): tx = threadIdx.x, out_y = threadIdx.y; here threads 0..127 (s_desc_notile.cu:33-86)
                if (threadIdx.x < 128) {
                    const int tx = threadIdx.x & 31, out_y = threadIdx.x >> 5;
                    const int in_x = tx & 7;
                    const float stepbase = -2.5f + 1.0f / 16.0f;
                    float dpt[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                    for (int xoff = 0; xoff < 2; ++xoff) {
                        const int xd = (xoff << 3) + in_x;
                        const int newx = (xoff << 3) + tx;
                        for (int yoff = 0; yoff < 2; ++yoff)
                            for (int in_y = 0; in_y < 8; ++in_y) {
                                const int yd = (yoff << 3) + in_y;
                                const int newy = (out_y << 3) + yd;
                                const float wgt = c_desc_tile[xd] * c_desc_tile[yd];
                                const float stepx = stepbase + scalbnf((float)newx, -3);
                                const float stepy = stepbase + scalbnf((float)newy, -3);
                                const float ptx = cos_t * stepx + -sin_t * stepy;
                                const float pty = cos_t * stepy + sin_t * stepx;
                                float mod, th;
                                gradient_rot(pl, x + ptx * SBP, y + pty * SBP, cos_t, sin_t, mod, th);
                                th += (th < 0.0f ? kPi2d : 0.0f);
                                const float tth = th * k4RPi;
                                const int fo = (int)floorf(th * k4RPi);
                                const float do0 = tth - (float)fo;
                                const int fo0 = fo & 7, fo1 = (fo0 + 1) & 7;
                                const float ww = c_desc_gauss[newy * 40 + newx] * mod;
                                const float ox = (1.0f - do0) * ww, oy = do0 * ww;
#pragma unroll
                                for (int b = 0; b < 8; ++b) {
                                    if (fo0 == b) dpt[b] += wgt * ox;
                                }
#pragma unroll
                                for (int b = 0; b < 8; ++b) {
                                    if (fo1 == b) dpt[b] += wgt * oy;
                                }
                            }
                    }
                    float mine = 0.0f;
#pragma unroll
                    for (int b = 0; b < 8; ++b) {
                        dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 4, 8);
                        dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 2, 8);
                        dpt[b] += __shfl_down_sync(0xffffffffu, dpt[b], 1, 8);
                        dpt[b] = __shfl_sync(0xffffffffu, dpt[b], 0, 8);
                        if (in_x == b) mine = dpt[b];
                    }
                    raw[out_y * 32 + tx] = mine;
                }
            }
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            float4 v = *reinterpret_cast<const float4*>(raw + 4 * lane);
            v = normalize_descriptor(v, lane, k.norm_mode, k.norm_multi);
            reinterpret_cast<float4*>(desc[d].features)[lane] = v;
        }
        __syncthreads();
    }
}

// desc_gauss / desc_tile exactly as the reference's host code fills them (sift_constants.cu:34-48)
void ensure_tables()
{
    static std::mutex mu;
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    if (dev < 0 || dev >= 64 || done[dev]) return;
    float gauss[40 * 40], tile[16];
    const float dn_step = 1.0f / 8.0f;
    const float dn_base = 0.5f * dn_step - 20.0f * dn_step;
    for (int y = 0; y < 40; ++y)
        for (int x = 0; x < 40; ++x) {
            const float dnx = dn_base + x * dn_step, dny = dn_base + y * dn_step;
            gauss[y * 40 + x] = expf(-scalbnf(dnx * dnx + dny * dny, -3));
        }
    for (int i = 0; i < 16; ++i) {
        const float nx = -1.0f + 1.0f / 16.0f + i * 1.0f / 8.0f;
        tile[i] = 1.0f - fabs(nx);
    }
    cudaMemcpyToSymbol(c_desc_gauss, gauss, sizeof(gauss));
    cudaMemcpyToSymbol(c_desc_tile, tile, sizeof(tile));
    done[dev] = true;
}

} // namespace

int launch_descriptors_mode(int mode, const PyramidView& pyr, const Consts& k, const ps_extremum* ext, const int* feat_to_ext,
                            ps_descriptor* desc, Counters* ct, cudaStream_t st)
{
    ensure_tables();
    const int grid = sm_count() * 8;
    switch (mode) {
        case PS_DESC_GRID:   desc_mode_kernel<PS_DESC_GRID><<<grid, MT, 0, st>>>(pyr, k, ext, feat_to_ext, desc, ct); break;
        case PS_DESC_IGRID:  desc_mode_kernel<PS_DESC_IGRID><<<grid, MT, 0, st>>>(pyr, k, ext, feat_to_ext, desc, ct); break;
        case PS_DESC_ILOOP:  desc_mode_kernel<PS_DESC_ILOOP><<<grid, MT, 0, st>>>(pyr, k, ext, feat_to_ext, desc, ct); break;
        case PS_DESC_NOTILE: desc_mode_kernel<PS_DESC_NOTILE><<<grid, MT, 0, st>>>(pyr, k, ext, feat_to_ext, desc, ct); break;
        default: return -1;
    }
    return 1;
}

} // namespace psb
