// C-ABI layer: the stateless batched entry points, ps_match .. ps_mesh_texture.  Each checks its arguments, sets the
// device, calls its run_* and finishes.  The argument rules several of them share are written once below; where each
// check sits relative to set_device is part of the entry point's behaviour (tests/test_abi_host_checks_cpu.py).
#include "ps_internal.h"
#include "popsift_b200_guided.h"
#include "popsift_b200_retrieval.h"

#include <algorithm>
#include <cstring>
#include <initializer_list>
#include <string>
#include <vector>

using namespace psb;

namespace {

bool set_device(int device)
{
    if (cudaSetDevice(device) == cudaSuccess) return true;
    cudaGetLastError();
    return false;
}

// every pointer is device memory on `device`
bool on_device(int device, std::initializer_list<const void*> ptrs)
{
    for (const void* p : ptrs)
        if (ps_pointer_device(p) != device) return false;
    return true;
}

// every entry of a host array of n device pointers on `device`
template <class T>
bool device_arrays(int device, T* const* p, int n)
{
    if (!p) return false;
    for (int j = 0; j < n; ++j)
        if (ps_pointer_device(p[j]) != device) return false;
    return true;
}

// a pinhole camera: finite, fx > 0 and fy > 0
bool camera_ok(const ps_camera& c)
{
    return std::isfinite(c.fx) && c.fx > 0.0f && std::isfinite(c.fy) && c.fy > 0.0f && std::isfinite(c.cx) && std::isfinite(c.cy);
}

// a row-major rotation: finite entries, max |R^T R - I| <= 1e-6 and det R > 0
bool rotation_ok(const double* R)
{
    for (int i = 0; i < 9; ++i)
        if (!std::isfinite(R[i])) return false;
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            const double d = R[a] * R[b] + R[3 + a] * R[3 + b] + R[6 + a] * R[6 + b] - (a == b ? 1.0 : 0.0);
            if (!(std::fabs(d) <= 1e-6)) return false;
        }
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    return det > 0.0;
}

// a pose: a rotation and a finite t
bool rigid_ok(const ps_rigid& p)
{
    return rotation_ok(p.R) && std::isfinite(p.t[0]) && std::isfinite(p.t[1]) && std::isfinite(p.t[2]);
}

// an image's geometry: min_side .. 65535 pixels a side, rows at least as wide as the image
bool image_ok(const ps_image& im, int min_side)
{
    return !(im.width < min_side || im.height < min_side || im.width > 65535 || im.height > 65535 || im.pitch < im.width);
}

// a correspondence CSR: both arrays given, no start or count negative; *rows = the largest end
bool corr_rows(int n_pairs, const int32_t* corr_start, const int32_t* n_corr, int64_t* rows)
{
    if (!corr_start || !n_corr) return false;
    *rows = 0;
    for (int p = 0; p < n_pairs; ++p) {
        if (corr_start[p] < 0 || n_corr[p] < 0) return false;
        *rows = std::max<int64_t>(*rows, (int64_t)corr_start[p] + n_corr[p]);
    }
    return true;
}

// RANSAC parameters: 1 .. 65536 samples, a finite threshold > 0, refine 0 or 1
bool ransac_ok(int n_samples, float threshold, int refine)
{
    return n_samples >= 1 && n_samples <= 65536 && std::isfinite(threshold) && threshold > 0.0f && (refine == 0 || refine == 1);
}

// the parameters bundle adjustment, rotation averaging and positioning share: a PS_LOSS_* with a finite scale > 0,
// 0 .. 10000 iterations, 1 .. 10000 CG iterations and a CG tolerance in [0, 1)
bool solver_ok(int loss, double loss_scale, int max_iters, int cg_max_iters, double cg_tol)
{
    return loss >= PS_LOSS_SQUARED && loss <= PS_LOSS_CAUCHY && max_iters >= 0 && max_iters <= 10000 && cg_max_iters >= 1 &&
           cg_max_iters <= 10000 && std::isfinite(loss_scale) && loss_scale > 0.0 && cg_tol >= 0.0 && cg_tol < 1.0;
}

// both ends of every pair a set index
bool pairs_in_range(int n_sets, const int32_t* pairs, int n_pairs)
{
    for (int p = 0; p < 2 * n_pairs; ++p)
        if (pairs[p] < 0 || pairs[p] >= n_sets) return false;
    return true;
}

// the per-set checks of the batched entry points: no negative count, and every non-empty set's pointer non-null, on
// `device` and aligned to align_mask + 1 bytes; *N (optional) = the pooled count
template <class T>
bool check_sets(int device, int n_sets, const int32_t* n_desc, const T* const* ptrs, uintptr_t align_mask, int64_t* N = nullptr)
{
    if (n_sets > 0 && (!n_desc || !ptrs)) return false;
    int64_t total = 0;
    for (int i = 0; i < n_sets; ++i) {
        if (n_desc[i] < 0) return false;
        if (n_desc[i] > 0 && (!ptrs[i] || (reinterpret_cast<uintptr_t>(ptrs[i]) & align_mask) || ps_pointer_device(ptrs[i]) != device))
            return false;
        total += n_desc[i];
    }
    if (N) *N = total;
    return true;
}

// set indices in range; *rows = the left sets' rows summed over the pairs; *work (optional): some pair has rows and a
// non-empty right set
bool check_pairs(int n_sets, const int32_t* n_desc, const int32_t* pairs, int n_pairs, int64_t* rows, bool* work = nullptr)
{
    *rows = 0;
    if (work) *work = false;
    if (!pairs_in_range(n_sets, pairs, n_pairs)) return false;
    for (int p = 0; p < n_pairs; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        *rows += n_desc[l];
        if (work) *work |= n_desc[l] > 0 && n_desc[r] > 0;
    }
    return true;
}

// what a run found wrong on the device, reported as "<name>: <what>"
constexpr const char* kBadEdge = "an edge endpoint is out of range";
constexpr const char* kBadMember = "a member id or d_track_start is out of range";
constexpr const char* kBadVertex = "a triangle's vertex index is out of range";

// the tail of every synchronous entry point: a run_* failure (launched < 0) keeps its message; an index the run found
// out of range (bad) is an argument error "<name>: <what>"; otherwise wait for the legacy stream and report what it
// returns as "<name>: <cuda error>"
int finish(const char* name, int launched, const char* err, bool bad = false, const char* what = nullptr)
{
    if (launched < 0) { set_last_error(err ? err : std::string(name) + " failed"); return PS_ERR_CUDA; }
    if (bad) { set_last_error(std::string(name) + ": " + what); return PS_ERR_ARG; }
    const cudaError_t e = cudaStreamSynchronize(nullptr);
    if (e != cudaSuccess) { set_last_error(std::string(name) + ": " + cudaGetErrorString(e)); cudaGetLastError(); return PS_ERR_CUDA; }
    return PS_OK;
}

} // namespace

extern "C" int ps_match(int device, const ps_descriptor* d_left, int n_left, const ps_descriptor* d_right, int n_right,
                        int32_t* d_out, int flags)
{
    if (n_left < 0 || n_right < 0 || (n_left > 0 && (!d_left || !d_out)) || (n_right > 0 && !d_right)) return PS_ERR_ARG;
    if (n_left == 0) return PS_OK;
    if (!set_device(device)) return PS_ERR_CUDA;
    const char* err = nullptr;
    const int n = run_match(d_left, n_left, d_right, n_right, d_out, flags, nullptr, &err);
    return finish("ps_match", n, err);
}

extern "C" int ps_match_batch(int device, int n_sets, const ps_descriptor* const* d_sets, const int32_t* n_desc,
                              int n_pairs, const int32_t* pairs, int32_t* d_out, int flags)
{
    if (n_sets < 0 || n_pairs < 0 || (n_sets > 0 && (!d_sets || !n_desc)) || (n_pairs > 0 && !pairs)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t rows = 0;
    if (!check_sets(device, n_sets, n_desc, d_sets, 0) || !check_pairs(n_sets, n_desc, pairs, n_pairs, &rows)) return PS_ERR_ARG;
    if (rows == 0) return PS_OK;
    if (!d_out) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_match_batch(d_sets, n_desc, n_sets, pairs, n_pairs, d_out, flags, nullptr, &err);
    return finish("ps_match_batch", n, err);
}

extern "C" int ps_descriptors_to_u8(int device, const ps_descriptor* d_in, int n, uint8_t* d_out)
{
    if (n < 0 || (n > 0 && (!d_in || !d_out))) return PS_ERR_ARG;
    if (n == 0) return PS_OK;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!on_device(device, {d_in, d_out})) return PS_ERR_ARG;
    return finish("ps_descriptors_to_u8", run_descriptors_to_u8(d_in, n, d_out, nullptr), nullptr);
}

extern "C" int ps_match_u8_batch(int device, int n_sets, const uint8_t* const* d_sets, const int32_t* n_desc,
                                 int n_pairs, const int32_t* pairs, int32_t* d_out, int flags)
{
    if (n_sets < 0 || n_pairs < 0 || (n_sets > 0 && (!d_sets || !n_desc)) || (n_pairs > 0 && !pairs)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t rows = 0;
    if (!check_sets(device, n_sets, n_desc, d_sets, 15u) || !check_pairs(n_sets, n_desc, pairs, n_pairs, &rows)) return PS_ERR_ARG;
    if (rows == 0) return PS_OK;
    if (!d_out) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_match_u8_batch(d_sets, n_desc, n_sets, pairs, n_pairs, d_out, flags, nullptr, &err);
    return finish("ps_match_u8_batch", n, err);
}

extern "C" int ps_match_correspondences(int device, int n_sets, const ps_feature* const* d_feat, const int32_t* const* d_rev,
                                        const int32_t* n_desc, int n_pairs, const int32_t* pairs, const int32_t* d_match,
                                        float* d_corr, int32_t* d_src, int32_t* n_corr)
{
    if (n_sets < 0 || n_pairs < 0 || (n_sets > 0 && (!d_feat || !d_rev || !n_desc)) || (n_pairs > 0 && (!pairs || !n_corr))) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t rows = 0;
    if (!check_sets(device, n_sets, n_desc, d_feat, 0) || !check_sets(device, n_sets, n_desc, d_rev, 0) ||
        !check_pairs(n_sets, n_desc, pairs, n_pairs, &rows))
        return PS_ERR_ARG;
    if (rows == 0) {
        for (int p = 0; p < n_pairs; ++p) n_corr[p] = 0;
        return PS_OK;
    }
    if (rows > 0x7fffffff) return PS_ERR_ARG;
    if (!on_device(device, {d_match, d_corr, d_src})) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_match_correspondences(d_feat, d_rev, n_desc, pairs, n_pairs, d_match, d_corr, d_src, n_corr, nullptr, &err);
    return finish("ps_match_correspondences", n, err);
}

extern "C" int ps_verify_batch(int device, int n_pairs, const float* d_corr, const int32_t* corr_start, const int32_t* n_corr,
                               const ps_verify_params* prm, float* d_models, int32_t* d_n_inliers, uint8_t* d_inlier_mask,
                               const ps_verify_taps* taps)
{
    if (n_pairs < 0 || !prm) return PS_ERR_ARG;
    if (prm->model != PS_GEOM_HOMOGRAPHY && prm->model != PS_GEOM_FUNDAMENTAL) return PS_ERR_ARG;
    if (!ransac_ok(prm->n_samples, prm->threshold, prm->refine)) return PS_ERR_ARG;
    if (n_pairs == 0) return PS_OK;
    int64_t rows = 0;
    if (!corr_rows(n_pairs, corr_start, n_corr, &rows)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!on_device(device, {d_models, d_n_inliers})) return PS_ERR_ARG;
    if (rows > 0 && (!on_device(device, {d_corr, d_inlier_mask}) || (reinterpret_cast<uintptr_t>(d_corr) & 15u))) return PS_ERR_ARG;
    if (taps && !on_device(device, {taps->d_counts, taps->d_models})) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_verify_batch(n_pairs, d_corr, corr_start, n_corr, *prm, d_models, d_n_inliers, d_inlier_mask, taps, nullptr, &err);
    return finish("ps_verify_batch", n, err);
}

extern "C" int ps_relative_pose_batch(int device, int n_pairs, const float* d_corr, const int32_t* corr_start, const int32_t* n_corr,
                                      const ps_camera* cams, const ps_pose_params* prm, ps_two_view* d_out, uint8_t* d_inlier_mask,
                                      float* d_points, const ps_verify_taps* taps)
{
    if (n_pairs < 0 || !prm) return PS_ERR_ARG;
    if (!ransac_ok(prm->n_samples, prm->threshold, prm->refine)) return PS_ERR_ARG;
    if (n_pairs == 0) return PS_OK;
    int64_t rows = 0;
    if (!cams || !corr_rows(n_pairs, corr_start, n_corr, &rows)) return PS_ERR_ARG;
    for (int k = 0; k < 2 * n_pairs; ++k)
        if (!camera_ok(cams[k])) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (ps_pointer_device(d_out) != device) return PS_ERR_ARG;
    if (d_points && ps_pointer_device(d_points) != device) return PS_ERR_ARG;
    if (rows > 0 && (!on_device(device, {d_corr, d_inlier_mask}) || (reinterpret_cast<uintptr_t>(d_corr) & 15u))) return PS_ERR_ARG;
    if (taps && !on_device(device, {taps->d_counts, taps->d_models})) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_relative_pose_batch(n_pairs, d_corr, corr_start, n_corr, cams, *prm, d_out, d_inlier_mask, d_points, taps, nullptr, &err);
    return finish("ps_relative_pose_batch", n, err);
}

// both guided entry points: the argument checks of ps_match_batch / ps_match_u8_batch and ps_match_correspondences, the
// model and threshold, and d_models when some pair has rows and a non-empty right set; then the run
static int match_guided(const char* name, bool u8, int device, int n_sets, const void* const* d_sets, const ps_feature* const* d_feat,
                        const int32_t* const* d_rev, const int32_t* n_desc, int n_pairs, const int32_t* pairs,
                        const float* d_models, int model, float threshold, int32_t* d_out, int flags)
{
    if (n_sets < 0 || n_pairs < 0 || (n_sets > 0 && (!d_sets || !d_feat || !d_rev || !n_desc)) || (n_pairs > 0 && !pairs)) return PS_ERR_ARG;
    if (model != PS_GEOM_HOMOGRAPHY && model != PS_GEOM_FUNDAMENTAL) return PS_ERR_ARG;
    if (!std::isfinite(threshold) || !(threshold > 0.0f)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t rows = 0;
    bool work = false;
    if (!check_sets(device, n_sets, n_desc, d_sets, u8 ? 15u : 0u) || !check_sets(device, n_sets, n_desc, d_feat, 0) ||
        !check_sets(device, n_sets, n_desc, d_rev, 0) || !check_pairs(n_sets, n_desc, pairs, n_pairs, &rows, &work))
        return PS_ERR_ARG;
    if (rows == 0) return PS_OK;
    if (!d_out) return PS_ERR_ARG;
    if (work && ps_pointer_device(d_models) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = u8 ? run_match_u8_guided_batch(reinterpret_cast<const uint8_t* const*>(d_sets), d_feat, d_rev, n_desc, n_sets, pairs, n_pairs,
                                                 d_models, model, threshold, d_out, flags, nullptr, &err)
                     : run_match_guided_batch(reinterpret_cast<const ps_descriptor* const*>(d_sets), d_feat, d_rev, n_desc, n_sets, pairs,
                                              n_pairs, d_models, model, threshold, d_out, flags, nullptr, &err);
    return finish(name, n, err);
}

extern "C" int ps_match_guided_batch(int device, int n_sets, const ps_descriptor* const* d_sets, const ps_feature* const* d_feat,
                                     const int32_t* const* d_rev, const int32_t* n_desc, int n_pairs, const int32_t* pairs,
                                     const float* d_models, int model, float threshold, int32_t* d_out, int flags)
{
    return match_guided("ps_match_guided_batch", false, device, n_sets, reinterpret_cast<const void* const*>(d_sets), d_feat, d_rev,
                        n_desc, n_pairs, pairs, d_models, model, threshold, d_out, flags);
}

extern "C" int ps_match_u8_guided_batch(int device, int n_sets, const uint8_t* const* d_sets, const ps_feature* const* d_feat,
                                        const int32_t* const* d_rev, const int32_t* n_desc, int n_pairs, const int32_t* pairs,
                                        const float* d_models, int model, float threshold, int32_t* d_out, int flags)
{
    return match_guided("ps_match_u8_guided_batch", true, device, n_sets, reinterpret_cast<const void* const*>(d_sets), d_feat, d_rev,
                        n_desc, n_pairs, pairs, d_models, model, threshold, d_out, flags);
}

extern "C" int ps_vlad_train(int device, int n_sets, const ps_descriptor* const* d_sets, const int32_t* n_desc, int k, int iters,
                             uint64_t seed, float* d_centroids, int flags)
{
    if (n_sets < 0 || k < 1 || k > 1024 || iters < 0 || iters > 1000) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0;
    if (!check_sets(device, n_sets, n_desc, d_sets, 0, &N) || N < k || N >= 0x80000000LL) return PS_ERR_ARG;
    if (ps_pointer_device(d_centroids) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_vlad_train(d_sets, n_desc, n_sets, k, iters, seed, d_centroids, flags, nullptr, &err);
    return finish("ps_vlad_train", n, err);
}

extern "C" int ps_vlad_encode(int device, int n_sets, const ps_descriptor* const* d_sets, const int32_t* n_desc, int k,
                              const float* d_centroids, float* d_vlad, int32_t* d_assign, int flags)
{
    if (n_sets < 0 || k < 1 || k > 1024) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0;
    if (!check_sets(device, n_sets, n_desc, d_sets, 0, &N)) return PS_ERR_ARG;
    if (n_sets == 0) return PS_OK;
    if (N >= 0x80000000LL) return PS_ERR_ARG;
    if (!on_device(device, {d_centroids, d_vlad})) return PS_ERR_ARG;
    if (d_assign && N > 0 && ps_pointer_device(d_assign) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    const int n = run_vlad_encode(d_sets, n_desc, n_sets, k, d_centroids, d_vlad, d_assign, flags, nullptr, &err);
    return finish("ps_vlad_encode", n, err);
}

extern "C" int ps_retrieve_pairs(int device, int n, const float* d_vec, int dim, int m, int32_t* d_nbr, float* d_score)
{
    if (n < 0 || dim <= 0 || (dim & 3) || m < 1 || m > 128) return PS_ERR_ARG;
    if (n == 0) return PS_OK;
    if ((int64_t)n * m >= 0x80000000LL) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (reinterpret_cast<uintptr_t>(d_vec) & 15u) return PS_ERR_ARG;
    if (!on_device(device, {d_vec, d_nbr, d_score})) return PS_ERR_ARG;
    const char* err = nullptr;
    const int r = run_retrieve_pairs(n, d_vec, dim, m, d_nbr, d_score, nullptr, &err);
    return finish("ps_retrieve_pairs", r, err);
}

// both track entry points: the feature counts (none negative, N < 2^31), min_length, counts and the outputs; *N = the
// number of features
static bool check_tracks(int device, int n_sets, const int32_t* n_feat, int min_length, const int32_t* d_track_of,
                         const int32_t* d_track_start, const int32_t* d_members, const ps_track_counts* counts, int64_t* N)
{
    if (n_sets < 0 || (n_sets > 0 && !n_feat) || min_length < 2 || !counts) return false;
    *N = 0;
    for (int i = 0; i < n_sets; ++i) {
        if (n_feat[i] < 0) return false;
        *N += n_feat[i];
    }
    if (*N >= 0x80000000LL) return false;
    if (ps_pointer_device(d_track_start) != device) return false;
    return *N == 0 || on_device(device, {d_track_of, d_members});
}

extern "C" int ps_tracks_from_edges(int device, int n_sets, const int32_t* n_feat, int n_edges, const int32_t* d_edges, int min_length,
                                    int32_t* d_track_of, int32_t* d_track_start, int32_t* d_members, ps_track_counts* counts)
{
    if (n_edges < 0 || (n_edges > 0 && !d_edges)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0;
    if (!check_tracks(device, n_sets, n_feat, min_length, d_track_of, d_track_start, d_members, counts, &N)) return PS_ERR_ARG;
    if (n_edges > 0 && ps_pointer_device(d_edges) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    bool bad = false;
    const int n = run_tracks_from_edges(n_sets, n_feat, n_edges, d_edges, min_length, d_track_of, d_track_start, d_members, counts,
                                        &bad, nullptr, &err);
    return finish("ps_tracks_from_edges", n, err, bad, kBadEdge);
}

extern "C" int ps_tracks_from_matches(int device, int n_sets, const int32_t* n_feat, const int32_t* const* d_rev, const int32_t* n_desc,
                                      int n_pairs, const int32_t* pairs, const int32_t* d_match, const int32_t* d_src, const int32_t* n_corr,
                                      const uint8_t* d_inlier_mask, int min_length, int32_t* d_track_of, int32_t* d_track_start,
                                      int32_t* d_members, ps_track_counts* counts)
{
    if (n_sets < 0 || n_pairs < 0 || (n_sets > 0 && (!d_rev || !n_desc)) || (n_pairs > 0 && (!pairs || !n_corr))) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0, rows = 0;
    if (!check_tracks(device, n_sets, n_feat, min_length, d_track_of, d_track_start, d_members, counts, &N) ||
        !check_sets(device, n_sets, n_desc, d_rev, 0) || !check_pairs(n_sets, n_desc, pairs, n_pairs, &rows))
        return PS_ERR_ARG;
    if (rows > 0x7fffffff) return PS_ERR_ARG;
    std::vector<int32_t> off(n_sets + 1, 0);
    for (int i = 0; i < n_sets; ++i) off[i + 1] = off[i] + n_feat[i];
    std::vector<TrackPair> tp(n_pairs);
    int64_t row0 = 0, corr = 0;
    for (int p = 0; p < n_pairs; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        if (n_corr[p] < 0 || n_corr[p] > n_desc[l]) return PS_ERR_ARG;
        tp[p] = TrackPair{0, row0, d_rev[l], d_rev[r], off[l], off[r], n_desc[l], n_desc[r], n_feat[l], n_feat[r], n_corr[p], 0};
        row0 += n_desc[l];
        corr += n_corr[p];
    }
    if (corr > 0 && (!on_device(device, {d_match, d_src}) || (d_inlier_mask && ps_pointer_device(d_inlier_mask) != device)))
        return PS_ERR_ARG;
    const char* err = nullptr;
    bool bad = false;
    const int n = run_tracks_from_matches(n_sets, n_feat, tp, d_match, d_src, d_inlier_mask, min_length, d_track_of, d_track_start,
                                          d_members, counts, &bad, nullptr, &err);
    return finish("ps_tracks_from_matches", n, err, bad, kBadEdge);
}

// the host checks ps_triangulate_tracks and ps_bundle_adjust share: the counts, the cameras and the poses
static bool check_tracks_call(int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                              const ps_rigid* poses, int n_tracks, int n_members)
{
    if (n_sets < 0 || n_tracks < 0 || n_members < 0) return false;
    if (n_sets > 0 && (!n_feat || !d_feat || !cams || !poses)) return false;
    for (int i = 0; i < n_sets; ++i)
        if (!camera_ok(cams[i]) || !rigid_ok(poses[i])) return false;
    return true;
}

extern "C" int ps_triangulate_tracks(int device, int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                                     const ps_rigid* poses, int n_tracks, const int32_t* d_track_start, const int32_t* d_members, int n_members,
                                     const ps_triangulate_params* prm, ps_track_point* d_points, uint8_t* d_obs_mask, float* d_obs_error,
                                     ps_triangulate_counts* counts)
{
    if (!prm || !counts || !check_tracks_call(n_sets, n_feat, d_feat, cams, poses, n_tracks, n_members)) return PS_ERR_ARG;
    if (!std::isfinite(prm->max_error) || !(prm->max_error > 0.0f)) return PS_ERR_ARG;
    if (!(prm->min_angle >= 0.0f && prm->min_angle < 90.0f)) return PS_ERR_ARG;
    if (prm->min_views < 2 || prm->n_samples < 1 || prm->n_samples > 65536 || prm->refine_iters < 0 || prm->refine_iters > 32) return PS_ERR_ARG;
    if (n_tracks == 0) {
        std::memset(counts, 0, sizeof(*counts));
        return PS_OK;
    }
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0;
    if (!check_sets(device, n_sets, n_feat, d_feat, 0, &N) || N >= 0x80000000LL) return PS_ERR_ARG;
    if (!on_device(device, {d_track_start, d_points})) return PS_ERR_ARG;
    if (n_members > 0 && !on_device(device, {d_members, d_obs_mask})) return PS_ERR_ARG;
    if (d_obs_error && ps_pointer_device(d_obs_error) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    bool bad = false;
    const int n = run_triangulate_tracks(n_sets, n_feat, d_feat, cams, poses, n_tracks, d_track_start, d_members, n_members, *prm, d_points,
                                         d_obs_mask, d_obs_error, counts, &bad, nullptr, &err);
    return finish("ps_triangulate_tracks", n, err, bad, kBadMember);
}

extern "C" int ps_bundle_adjust(int device, int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                                const ps_rigid* poses_in, int n_tracks, const int32_t* d_track_start, const int32_t* d_members, int n_members,
                                ps_track_point* d_points, const uint8_t* d_obs_mask, const uint8_t* fixed, const ps_bundle_params* prm,
                                ps_rigid* poses_out, float* d_obs_error, ps_bundle_report* report)
{
    if (!prm || !report || !poses_out || !fixed) return PS_ERR_ARG;
    if (!check_tracks_call(n_sets, n_feat, d_feat, cams, poses_in, n_tracks, n_members)) return PS_ERR_ARG;
    if (!solver_ok(prm->loss, prm->loss_scale, prm->max_iters, prm->cg_max_iters, prm->cg_tol)) return PS_ERR_ARG;
    if (!std::isfinite(prm->function_tol) || !(prm->function_tol >= 0.0)) return PS_ERR_ARG;
    if (!(prm->initial_lambda > 0.0 && prm->initial_lambda <= 1e32)) return PS_ERR_ARG;
    if (prm->scale_set < -1 || prm->scale_set >= n_sets || prm->scale_axis < 0 || prm->scale_axis > 2) return PS_ERR_ARG;
    bool any_fixed = false;
    for (int i = 0; i < n_sets; ++i) {
        if (fixed[i] > 1) return PS_ERR_ARG;
        any_fixed |= fixed[i] == 1;
    }
    if (!any_fixed) return PS_ERR_ARG;
    if (n_tracks == 0) {
        std::memset(report, 0, sizeof(*report));
        report->termination = PS_BA_NO_OBSERVATIONS;
        if (poses_out != poses_in) std::memcpy(poses_out, poses_in, (size_t)n_sets * sizeof(ps_rigid));
        return PS_OK;
    }
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0;
    if (!check_sets(device, n_sets, n_feat, d_feat, 0, &N) || N >= 0x80000000LL) return PS_ERR_ARG;
    if (!on_device(device, {d_track_start, d_points})) return PS_ERR_ARG;
    if (n_members > 0 && !on_device(device, {d_members, d_obs_mask})) return PS_ERR_ARG;
    if (d_obs_error && ps_pointer_device(d_obs_error) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    bool bad = false;
    std::vector<ps_rigid> out(n_sets);
    ps_bundle_report rep{};
    const int n = run_bundle_adjust(n_sets, n_feat, d_feat, cams, poses_in, n_tracks, d_track_start, d_members, n_members, d_points, d_obs_mask,
                                    fixed, *prm, out.data(), d_obs_error, &rep, &bad, nullptr, &err);
    const int rc = finish("ps_bundle_adjust", n, err, bad, kBadMember);
    if (rc == PS_OK) {
        std::memcpy(poses_out, out.data(), (size_t)n_sets * sizeof(ps_rigid));
        *report = rep;
    }
    return rc;
}

extern "C" int ps_rotation_averaging(int device, int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view,
                                     const ps_rotation_params* prm, double* R_out, uint8_t* registered, float* pair_error,
                                     ps_rotation_report* report)
{
    if (n_sets < 0 || n_pairs < 0 || !prm || !R_out || !registered || !report || (n_pairs > 0 && !pairs)) return PS_ERR_ARG;
    if (!pairs_in_range(n_sets, pairs, n_pairs)) return PS_ERR_ARG;
    if (!solver_ok(prm->loss, prm->loss_scale, prm->max_iters, prm->cg_max_iters, prm->cg_tol) || prm->min_inliers < 0) return PS_ERR_ARG;
    if (!std::isfinite(prm->step_tol) || !(prm->step_tol >= 0.0)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (n_pairs > 0 && ps_pointer_device(d_two_view) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    std::vector<double> R((size_t)n_sets * 9);
    std::vector<uint8_t> reg(n_sets);
    std::vector<float> perr(n_pairs);
    ps_rotation_report rep{};
    const int n = run_rotation_averaging(n_sets, n_pairs, pairs, d_two_view, *prm, R.data(), reg.data(), perr.data(), &rep, nullptr, &err);
    const int rc = finish("ps_rotation_averaging", n, err);
    if (rc == PS_OK) {
        if (n_sets) std::memcpy(R_out, R.data(), R.size() * 8);
        if (n_sets) std::memcpy(registered, reg.data(), reg.size());
        if (pair_error && n_pairs) std::memcpy(pair_error, perr.data(), perr.size() * 4);
        *report = rep;
    }
    return rc;
}

extern "C" int ps_global_positioning(int device, int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                                     const double* R, const uint8_t* registered, int n_tracks, const int32_t* d_track_start,
                                     const int32_t* d_members, int n_members, const ps_position_params* prm, ps_rigid* poses_out,
                                     uint8_t* positioned, double* d_X, ps_position_report* report)
{
    if (!prm || !report || n_sets < 0 || n_tracks < 0 || n_members < 0) return PS_ERR_ARG;
    if (n_sets > 0 && (!n_feat || !d_feat || !cams || !R || !registered || !poses_out || !positioned)) return PS_ERR_ARG;
    for (int i = 0; i < n_sets; ++i)
        if (!camera_ok(cams[i]) || !rotation_ok(R + 9 * (size_t)i) || registered[i] > 1) return PS_ERR_ARG;
    if (!solver_ok(prm->loss, prm->loss_scale, prm->max_iters, prm->cg_max_iters, prm->cg_tol)) return PS_ERR_ARG;
    if (!std::isfinite(prm->function_tol) || !(prm->function_tol >= 0.0)) return PS_ERR_ARG;
    if (n_tracks == 0) {
        std::memset(report, 0, sizeof(*report));
        report->termination = PS_GP_NO_OBSERVATIONS;
        for (int i = 0; i < n_sets; ++i) {
            std::memcpy(poses_out[i].R, R + 9 * (size_t)i, sizeof(poses_out[i].R));
            poses_out[i].t[0] = poses_out[i].t[1] = poses_out[i].t[2] = 0.0;
            positioned[i] = 0;
        }
        return PS_OK;
    }
    if (!set_device(device)) return PS_ERR_CUDA;
    int64_t N = 0;
    if (!check_sets(device, n_sets, n_feat, d_feat, 0, &N) || N >= 0x80000000LL) return PS_ERR_ARG;
    if (ps_pointer_device(d_track_start) != device) return PS_ERR_ARG;
    if (n_members > 0 && ps_pointer_device(d_members) != device) return PS_ERR_ARG;
    if (d_X && ps_pointer_device(d_X) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    bool bad = false;
    std::vector<ps_rigid> out(n_sets);
    std::vector<uint8_t> pos(n_sets);
    ps_position_report rep{};
    const int n = run_global_positioning(n_sets, n_feat, d_feat, cams, R, registered, n_tracks, d_track_start, d_members, n_members, *prm,
                                         out.data(), pos.data(), d_X, &rep, &bad, nullptr, &err);
    const int rc = finish("ps_global_positioning", n, err, bad, kBadMember);
    if (rc == PS_OK) {
        if (n_sets) std::memcpy(poses_out, out.data(), (size_t)n_sets * sizeof(ps_rigid));
        if (n_sets) std::memcpy(positioned, pos.data(), pos.size());
        *report = rep;
    }
    return rc;
}

extern "C" int ps_view_graph_filter(int device, int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view,
                                    const ps_view_graph_params* prm, uint8_t* keep, ps_cycle_stats* stats, ps_two_view* d_kept,
                                    ps_view_graph_report* report)
{
    if (n_sets < 0 || n_pairs < 0 || !prm || !keep || !report || (n_pairs > 0 && !pairs)) return PS_ERR_ARG;
    if (!pairs_in_range(n_sets, pairs, n_pairs)) return PS_ERR_ARG;
    if (prm->min_inliers < 0 || prm->min_consistent < 0 || prm->keep_untested < 0 || prm->keep_untested > 1) return PS_ERR_ARG;
    if (!std::isfinite(prm->max_cycle_error) || !(prm->max_cycle_error >= 0.0)) return PS_ERR_ARG;
    if (!(prm->min_fraction >= 0.0 && prm->min_fraction <= 1.0)) return PS_ERR_ARG;
    // duplicates, in either order, in O(pairs + sets): the larger ends bucketed by the smaller end, then each bucket's
    // larger ends stamped with the bucket's set
    std::vector<int32_t> start(n_sets + 1, 0), larger(n_pairs), seen(n_sets, -1);
    for (int p = 0; p < n_pairs; ++p) ++start[std::min(pairs[2 * p], pairs[2 * p + 1]) + 1];
    for (int i = 0; i < n_sets; ++i) start[i + 1] += start[i];
    {
        std::vector<int32_t> fill(start.begin(), start.end() - 1);
        for (int p = 0; p < n_pairs; ++p)
            larger[fill[std::min(pairs[2 * p], pairs[2 * p + 1])]++] = std::max(pairs[2 * p], pairs[2 * p + 1]);
    }
    for (int a = 0; a < n_sets; ++a)
        for (int k = start[a]; k < start[a + 1]; ++k) {
            if (seen[larger[k]] == a) {
                set_last_error("ps_view_graph_filter: two pairs join the same two sets");
                return PS_ERR_ARG;
            }
            seen[larger[k]] = a;
        }
    if (!set_device(device)) return PS_ERR_CUDA;
    if (n_pairs > 0 && ps_pointer_device(d_two_view) != device) return PS_ERR_ARG;
    if (d_kept && ps_pointer_device(d_kept) != device) return PS_ERR_ARG;
    if (n_pairs == 0) {
        std::memset(report, 0, sizeof(*report));
        return PS_OK;
    }
    const char* err = nullptr;
    std::vector<uint8_t> kp(n_pairs);
    std::vector<ps_cycle_stats> cs(stats ? n_pairs : 0);
    ps_view_graph_report rep{};
    const int n = run_view_graph_filter(n_sets, n_pairs, pairs, d_two_view, *prm, kp.data(), stats ? cs.data() : nullptr, d_kept, &rep,
                                        nullptr, &err);
    const int rc = finish("ps_view_graph_filter", n, err);
    if (rc == PS_OK) {
        std::memcpy(keep, kp.data(), kp.size());
        if (stats) std::memcpy(stats, cs.data(), cs.size() * sizeof(ps_cycle_stats));
        *report = rep;
    }
    return rc;
}

// [lo, hi) byte ranges of device arguments; true when two of them intersect
static bool ranges_overlap(const void* a, size_t na, const void* b, size_t nb)
{
    if (!a || !b || na == 0 || nb == 0) return false;
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
    return a0 < b0 + nb && b0 < a0 + na;
}

extern "C" int ps_two_view_config_batch(int device, int n_pairs, const float* d_corr, const int32_t* corr_start, const int32_t* n_corr,
                                        const ps_camera* cams, const ps_two_view* d_essential, const uint8_t* d_essential_mask,
                                        const int32_t* d_f_inliers, const float* d_homography, const uint8_t* d_h_mask,
                                        const ps_two_view_config_params* prm, ps_two_view* d_out, uint8_t* d_out_mask, float* d_points,
                                        ps_two_view_info* info)
{
    if (n_pairs < 0 || !prm || !info) return PS_ERR_ARG;
    if (prm->min_inliers < 0 || !std::isfinite(prm->threshold) || !(prm->threshold > 0.0f)) return PS_ERR_ARG;
    for (const double r : {prm->min_ef_ratio, prm->max_h_ratio, prm->min_rotation_ratio})
        if (!(r >= 0.0 && r <= 1.0)) return PS_ERR_ARG;
    if (n_pairs == 0) return PS_OK;
    int64_t rows = 0;
    if (!cams || !corr_rows(n_pairs, corr_start, n_corr, &rows)) return PS_ERR_ARG;
    for (int k = 0; k < 2 * n_pairs; ++k)
        if (!camera_ok(cams[k])) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!on_device(device, {d_essential, d_f_inliers, d_homography, d_out})) return PS_ERR_ARG;
    if (d_points && ps_pointer_device(d_points) != device) return PS_ERR_ARG;
    if (rows > 0 && (!on_device(device, {d_corr, d_essential_mask, d_h_mask, d_out_mask}) || (reinterpret_cast<uintptr_t>(d_corr) & 15u)))
        return PS_ERR_ARG;
    // no output may overlap an input or another output
    const size_t P = (size_t)n_pairs, R = (size_t)rows;
    const std::pair<const void*, size_t> in[] = {{d_corr, 16 * R}, {d_essential, sizeof(ps_two_view) * P}, {d_essential_mask, R},
                                                 {d_f_inliers, 4 * P}, {d_homography, 36 * P}, {d_h_mask, R}};
    const std::pair<const void*, size_t> out[] = {{d_out, sizeof(ps_two_view) * P}, {d_out_mask, R}, {d_points, d_points ? 16 * R : 0}};
    for (int o = 0; o < 3; ++o) {
        for (const auto& i : in)
            if (ranges_overlap(out[o].first, out[o].second, i.first, i.second)) return PS_ERR_ARG;
        for (int o2 = o + 1; o2 < 3; ++o2)
            if (ranges_overlap(out[o].first, out[o].second, out[o2].first, out[o2].second)) return PS_ERR_ARG;
    }
    const char* err = nullptr;
    std::vector<ps_two_view_info> inf(n_pairs);
    const int n = run_two_view_config_batch(n_pairs, d_corr, corr_start, n_corr, cams, d_essential, d_essential_mask, d_f_inliers,
                                            d_homography, d_h_mask, *prm, d_out, d_out_mask, d_points, inf.data(), nullptr, &err);
    const int rc = finish("ps_two_view_config_batch", n, err);
    if (rc == PS_OK) std::memcpy(info, inf.data(), inf.size() * sizeof(ps_two_view_info));
    return rc;
}

// The checks ps_depth_maps and ps_depth_filter share (n_refs > 0, the device already set): the sets, the references and
// the source CSR; the images, cameras and poses of every set they use, each image at least min_side pixels a side
static bool check_depth_call(int device, int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs,
                             const int32_t* refs, const int32_t* src_start, const int32_t* src_sets, int min_side)
{
    if (n_sets < 0 || !images || !cams || !poses || !refs || !src_start) return false;
    if (src_start[0] != 0) return false;
    for (int j = 0; j < n_refs; ++j)
        if (src_start[j + 1] < src_start[j]) return false;
    if (src_start[n_refs] > 0 && !src_sets) return false;
    std::vector<uint8_t> used(n_sets, 0);
    for (int j = 0; j < n_refs; ++j) {
        const int r = refs[j];
        if (r < 0 || r >= n_sets || (used[r] & 1)) return false;
        used[r] |= 1;
    }
    for (int j = 0; j < n_refs; ++j)
        for (int s = src_start[j]; s < src_start[j + 1]; ++s) {
            const int i = src_sets[s];
            if (i < 0 || i >= n_sets || i == refs[j]) return false;
            used[i] |= 2;
        }
    for (int i = 0; i < n_sets; ++i)
        if (used[i] && (!image_ok(images[i], min_side) || ps_pointer_device(images[i].data) != device || !camera_ok(cams[i]) ||
                        !rigid_ok(poses[i])))
            return false;
    return true;
}

extern "C" int ps_depth_maps(int device, int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs,
                             const int32_t* refs, const float* ranges, const int32_t* src_start, const int32_t* src_sets,
                             const ps_depth_params* prm, float* const* d_depth, float* const* d_cost, uint8_t* const* d_n_src,
                             ps_depth_report* report)
{
    if (n_sets < 0 || n_refs < 0 || !prm || !report) return PS_ERR_ARG;
    if (prm->n_depths < 2 || prm->n_depths > 1024 || prm->radius < 1 || prm->radius > 7 || prm->top_k < 1 || prm->top_k > 32 ||
        prm->min_sources < 1 || prm->min_sources > 32)
        return PS_ERR_ARG;
    if (!(prm->max_cost > 0.0f && prm->max_cost <= 2.0f) || !std::isfinite(prm->min_var) || !(prm->min_var >= 0.0f)) return PS_ERR_ARG;
    if (n_refs == 0) {
        std::memset(report, 0, sizeof(*report));
        return PS_OK;
    }
    if (!ranges) return PS_ERR_ARG;
    for (int j = 0; j < n_refs; ++j) {
        const float lo = ranges[2 * j], hi = ranges[2 * j + 1];
        if (!std::isfinite(lo) || !std::isfinite(hi) || !(lo > 0.0f) || !(lo < hi)) return PS_ERR_ARG;
    }
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!check_depth_call(device, n_sets, images, cams, poses, n_refs, refs, src_start, src_sets, 2 * prm->radius + 1)) return PS_ERR_ARG;
    if (!device_arrays(device, d_depth, n_refs) || !device_arrays(device, d_cost, n_refs) || !device_arrays(device, d_n_src, n_refs))
        return PS_ERR_ARG;
    const char* err = nullptr;
    ps_depth_report rep{};
    const int n = run_depth_maps(n_sets, images, cams, poses, n_refs, refs, ranges, src_start, src_sets, *prm, d_depth, d_cost, d_n_src,
                                 &rep, nullptr, &err);
    const int rc = finish("ps_depth_maps", n, err);
    if (rc == PS_OK) *report = rep;
    return rc;
}

extern "C" int ps_depth_filter(int device, int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs,
                               const int32_t* refs, const int32_t* src_start, const int32_t* src_sets, const float* const* d_depth,
                               const ps_depth_filter_params* prm, uint8_t* const* d_n_consistent, ps_dense_point* d_points,
                               ps_depth_filter_report* report)
{
    if (n_sets < 0 || n_refs < 0 || !prm || !report) return PS_ERR_ARG;
    if (!std::isfinite(prm->max_reproj_error) || !(prm->max_reproj_error > 0.0f) || !std::isfinite(prm->max_depth_diff) ||
        !(prm->max_depth_diff > 0.0f) || prm->min_consistent < 1 || prm->min_consistent > 255)
        return PS_ERR_ARG;
    if (n_refs == 0) {
        std::memset(report, 0, sizeof(*report));
        return PS_OK;
    }
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!check_depth_call(device, n_sets, images, cams, poses, n_refs, refs, src_start, src_sets, 1)) return PS_ERR_ARG;
    if (!device_arrays(device, d_depth, n_refs) || !device_arrays(device, d_n_consistent, n_refs) || ps_pointer_device(d_points) != device)
        return PS_ERR_ARG;
    int64_t total = 0;
    for (int j = 0; j < n_refs; ++j) total += (int64_t)images[refs[j]].width * images[refs[j]].height;
    if (total >= 0x80000000LL) return PS_ERR_ARG;
    const char* err = nullptr;
    ps_depth_filter_report rep{};
    const int n = run_depth_filter(n_sets, images, cams, poses, n_refs, refs, src_start, src_sets, d_depth, *prm, d_n_consistent, d_points,
                                   &rep, nullptr, &err);
    const int rc = finish("ps_depth_filter", n, err);
    if (rc == PS_OK) *report = rep;
    return rc;
}

// a volume's geometry and arrays (the device already set): finite origin and voxel > 0, dimensions 2 .. 2048 with fewer
// than 2^31 grid points, three disjoint arrays of device memory on `device`
static bool volume_ok(int device, const ps_volume* vol)
{
    if (!vol) return false;
    for (double o : vol->origin)
        if (!std::isfinite(o)) return false;
    if (!std::isfinite(vol->voxel) || !(vol->voxel > 0.0)) return false;
    for (int d : {vol->nx, vol->ny, vol->nz})
        if (d < 2 || d > 2048) return false;
    const size_t n = (size_t)vol->nx * vol->ny * vol->nz;
    if (n >= 0x80000000ull) return false;
    const float* arr[3] = {vol->tsdf, vol->weight, vol->grey};
    for (int a = 0; a < 3; ++a) {
        if (ps_pointer_device(arr[a]) != device) return false;
        for (int b = a + 1; b < 3; ++b)
            if (ranges_overlap(arr[a], 4 * n, arr[b], 4 * n)) return false;
    }
    return true;
}

extern "C" int ps_volume_clear(int device, const ps_volume* vol)
{
    if (!vol) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!volume_ok(device, vol)) return PS_ERR_ARG;
    const char* err = nullptr;
    return finish("ps_volume_clear", run_volume_clear(*vol, nullptr, &err), err);
}

extern "C" int ps_tsdf_integrate(int device, int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses,
                                 const float* const* d_depth, const uint8_t* const* d_n_consistent, const ps_tsdf_params* prm,
                                 const ps_volume* vol, ps_tsdf_report* report)
{
    if (n_views < 0 || !prm || !vol || !report) return PS_ERR_ARG;
    if (!std::isfinite(prm->trunc) || !(prm->trunc > 0.0f) || prm->min_consistent < 0 || prm->min_consistent > 255) return PS_ERR_ARG;
    if (n_views > 0 && (!images || !cams || !poses || !d_depth || (prm->min_consistent > 0 && !d_n_consistent))) return PS_ERR_ARG;
    for (int v = 0; v < n_views; ++v)
        if (!image_ok(images[v], 1) || !camera_ok(cams[v]) || !rigid_ok(poses[v])) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!volume_ok(device, vol)) return PS_ERR_ARG;
    for (int v = 0; v < n_views; ++v) {
        if (!on_device(device, {images[v].data, d_depth[v]})) return PS_ERR_ARG;
        if (prm->min_consistent > 0 && ps_pointer_device(d_n_consistent[v]) != device) return PS_ERR_ARG;
    }
    if (n_views == 0) {
        std::memset(report, 0, sizeof(*report));
        return PS_OK;
    }
    const char* err = nullptr;
    ps_tsdf_report rep{};
    const int n = run_tsdf_integrate(n_views, images, cams, poses, d_depth, d_n_consistent, *prm, *vol, &rep, nullptr, &err);
    const int rc = finish("ps_tsdf_integrate", n, err);
    if (rc == PS_OK) *report = rep;
    return rc;
}

extern "C" int ps_tsdf_mesh(int device, const ps_volume* vol, const ps_mesh_params* prm, int64_t max_vertices, int64_t max_triangles,
                            ps_mesh_vertex* d_vertices, int32_t* d_triangles, ps_mesh_report* report)
{
    if (!vol || !prm || !report || max_vertices < 0 || max_triangles < 0) return PS_ERR_ARG;
    if (!std::isfinite(prm->min_weight) || !(prm->min_weight > 0.0f)) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    if (!volume_ok(device, vol)) return PS_ERR_ARG;
    if (max_vertices > 0 && ps_pointer_device(d_vertices) != device) return PS_ERR_ARG;
    if (max_triangles > 0 && ps_pointer_device(d_triangles) != device) return PS_ERR_ARG;
    const char* err = nullptr;
    ps_mesh_report rep{};
    bool overflow = false;
    const int n = run_tsdf_mesh(*vol, *prm, max_vertices, max_triangles, d_vertices, d_triangles, &rep, &overflow, nullptr, &err);
    const int rc = finish("ps_tsdf_mesh", n, err);
    if (rc != PS_OK) return rc;
    *report = rep;
    if (overflow) {
        set_last_error("ps_tsdf_mesh: the mesh does not fit the outputs' capacities");
        return PS_ERR_OVERFLOW;
    }
    return PS_OK;
}

// the counts and mesh arrays ps_mesh_render and ps_mesh_texture share (before the device is set)
static bool mesh_counts_ok(int n_views, int64_t n_vertices, int64_t n_triangles, const ps_mesh_vertex* d_vertices, const int32_t* d_triangles)
{
    if (n_views < 0 || n_vertices < 0 || n_triangles < 0 || n_triangles >= 0x80000000LL) return false;
    return n_triangles == 0 || (d_vertices && d_triangles);
}

extern "C" int ps_mesh_render(int device, int n_views, const int32_t* sizes, const ps_camera* cams, const ps_rigid* poses,
                              const ps_mesh_vertex* d_vertices, int64_t n_vertices, const int32_t* d_triangles, int64_t n_triangles,
                              const ps_render_params* prm, float* const* d_depth, int32_t* const* d_tri, ps_render_report* report)
{
    if (!prm || !report || !mesh_counts_ok(n_views, n_vertices, n_triangles, d_vertices, d_triangles)) return PS_ERR_ARG;
    if (!std::isfinite(prm->z_near) || !(prm->z_near > 0.0f)) return PS_ERR_ARG;
    if (n_views > 0 && (!sizes || !cams || !poses || !d_depth || !d_tri)) return PS_ERR_ARG;
    for (int v = 0; v < n_views; ++v) {
        if (sizes[2 * v] < 1 || sizes[2 * v] > 65535 || sizes[2 * v + 1] < 1 || sizes[2 * v + 1] > 65535) return PS_ERR_ARG;
        if (!camera_ok(cams[v]) || !rigid_ok(poses[v])) return PS_ERR_ARG;
    }
    if (!set_device(device)) return PS_ERR_CUDA;
    if (n_triangles > 0 && !on_device(device, {d_vertices, d_triangles})) return PS_ERR_ARG;
    if (!device_arrays(device, d_depth, n_views) && n_views > 0) return PS_ERR_ARG;
    if (!device_arrays(device, d_tri, n_views) && n_views > 0) return PS_ERR_ARG;
    if (n_views == 0) {
        std::memset(report, 0, sizeof(*report));
        return PS_OK;
    }
    const char* err = nullptr;
    ps_render_report rep{};
    bool bad = false;
    const int n = run_mesh_render(n_views, sizes, cams, poses, d_vertices, n_vertices, d_triangles, n_triangles, *prm, d_depth, d_tri, &rep,
                                  &bad, nullptr, &err);
    const int rc = finish("ps_mesh_render", n, err, bad, kBadVertex);
    if (rc == PS_OK) *report = rep;
    return rc;
}

extern "C" int ps_mesh_texture(int device, int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses,
                               const float* const* d_depth, const ps_mesh_vertex* d_vertices, int64_t n_vertices, const int32_t* d_triangles,
                               int64_t n_triangles, const ps_texture_params* prm, uint8_t* d_atlas, int32_t* d_view, ps_texture_report* report)
{
    if (!prm || !report || !mesh_counts_ok(n_views, n_vertices, n_triangles, d_vertices, d_triangles)) return PS_ERR_ARG;
    if (!std::isfinite(prm->z_near) || !(prm->z_near > 0.0f) || !std::isfinite(prm->depth_tol) || !(prm->depth_tol >= 0.0f) ||
        !(prm->min_cos >= 0.0f && prm->min_cos < 1.0f) || prm->cell < 3 || prm->cell > 64 || prm->cells_per_row < 1)
        return PS_ERR_ARG;
    if ((int64_t)prm->cells_per_row * prm->cell > 65535) return PS_ERR_ARG;
    if ((n_triangles + prm->cells_per_row - 1) / prm->cells_per_row * prm->cell > 65535) return PS_ERR_ARG;
    if (n_views > 0 && (!images || !cams || !poses || !d_depth)) return PS_ERR_ARG;
    if (n_triangles > 0 && (!d_atlas || !d_view)) return PS_ERR_ARG;
    for (int v = 0; v < n_views; ++v)
        if (!image_ok(images[v], 2) || !camera_ok(cams[v]) || !rigid_ok(poses[v])) return PS_ERR_ARG;
    if (!set_device(device)) return PS_ERR_CUDA;
    for (int v = 0; v < n_views; ++v)
        if (!on_device(device, {images[v].data, d_depth[v]})) return PS_ERR_ARG;
    if (n_triangles > 0 && !on_device(device, {d_vertices, d_triangles, d_atlas, d_view})) return PS_ERR_ARG;
    if (n_triangles == 0) {
        std::memset(report, 0, sizeof(*report));
        return PS_OK;
    }
    const char* err = nullptr;
    ps_texture_report rep{};
    bool bad = false;
    const int n = run_mesh_texture(n_views, images, cams, poses, d_depth, d_vertices, n_vertices, d_triangles, n_triangles, *prm, d_atlas,
                                   d_view, &rep, &bad, nullptr, &err);
    const int rc = finish("ps_mesh_texture", n, err, bad, kBadVertex);
    if (rc == PS_OK) *report = rep;
    return rc;
}
