/* Dense depth maps (an addition to the reference's interface): a depth for every pixel of posed images by a fronto-parallel
 * plane sweep with a zero-mean NCC window and best-K aggregation over source views, then a geometric-consistency check
 * between the depth maps of one call that keeps the consistent pixels as a world-space point cloud.
 *
 * The sparse chain ends with camera poses and a few thousand points per image (global poses, triangulation, bundle
 * adjustment).  The next step of every photogrammetry pipeline is dense reconstruction: AliceVision's DepthMap node and
 * COLMAP's patch_match_stereo follow their mappers.  These entry points take the 8-bit images where they already are on the
 * device, the pinhole cameras and the world-to-camera poses, and leave the depth maps and the points on the device.
 * Depth ranges and source views can be chosen from the tracks and their points (api.depth_ranges, api.select_sources).
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_DEPTH_H
#define POPSIFT_B200_DEPTH_H

#include "popsift_b200_triangulate.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_image {                 /* 24 bytes, HOST struct describing DEVICE pixels                            */
    const uint8_t* data;                  /* DEVICE, row-major grey levels                                             */
    int64_t pitch;                        /* bytes between rows, >= width                                              */
    int32_t width, height;
} ps_image;

typedef struct ps_depth_params {          /* 24 bytes */
    int32_t n_depths;                     /* planes, 2 .. 1024                                                         */
    int32_t radius;                       /* window half-size r, 1 .. 7: (2r+1)^2 pixels                               */
    int32_t top_k;                        /* source costs averaged, 1 .. 32                                            */
    int32_t min_sources;                  /* valid sources needed, 1 .. 32                                             */
    float   max_cost;                     /* a depth is kept when its cost <= max_cost, (0, 2]                         */
    float   min_var;                      /* window variance floor, grey levels^2, finite and >= 0                     */
} ps_depth_params;

typedef struct ps_depth_report {          /* 16 bytes, HOST */
    int64_t n_candidates;                 /* pixels whose window lies inside their reference image (step 4)            */
    int64_t n_depths;                     /* pixels with d_depth > 0                                                   */
} ps_depth_report;

typedef struct ps_depth_filter_params {   /* 16 bytes */
    float   max_reproj_error;             /* pixels, finite and > 0                                                    */
    float   max_depth_diff;               /* relative, finite and > 0                                                  */
    int32_t min_consistent;               /* 1 .. 255                                                                  */
    int32_t pad_;                         /* ignored                                                                   */
} ps_depth_filter_params;

typedef struct ps_dense_point {           /* 24 bytes, DEVICE */
    float    X[3];                        /* world coordinates (computed in double, rounded)                           */
    int32_t  ref;                         /* index into the call's ref list                                            */
    uint16_t x, y;                        /* the reference pixel                                                       */
    uint8_t  n_consistent;
    uint8_t  grey;                        /* the reference image's value at (x, y)                                     */
    uint16_t pad_;                        /* zero                                                                      */
} ps_dense_point;

typedef struct ps_depth_filter_report {   /* 16 bytes, HOST */
    int64_t n_tested;                     /* pixels with a depth > 0                                                   */
    int64_t n_points;                     /* records written to d_points                                               */
} ps_depth_filter_report;

/* One depth map per reference image.  Set i is the image images[i] (a HOST array of structs whose data is DEVICE memory),
 * with camera cams[i] and world-to-camera pose poses[i] (HOST, X_cam = R X + t).  refs[0 .. n_refs - 1] (HOST) are distinct
 * set ids; reference j has the depth range [ranges[2j], ranges[2j + 1]] (HOST floats) and the source sets
 * src_sets[src_start[j] .. src_start[j + 1] - 1] (HOST CSR, src_start[0] = 0, non-decreasing).  d_depth[j], d_cost[j] and
 * d_n_src[j] (HOST arrays of DEVICE pointers) hold w x h elements of reference j, row stride w.  The contract is stated in
 * real arithmetic; the device evaluates it in float (the homography, bilinear samples and box sums, with the samples and
 * the reference values taken minus 128, which changes no quantity below) and finishes each NCC in double.
 *   1. Pixels: pixel (column x, row y) is the point (x, y), the convention of the Feature records and ps_camera.
 *   2. Planes: iota_k = 1/d_min + k (1/d_max - 1/d_min) / (n - 1), k = 0 .. n - 1, n = n_depths; plane k is z = 1/iota_k in
 *      the reference camera frame.
 *   3. Warp: reference pixel p = (x, y) on plane k is the world point X = R_r^T (z K_r^-1 (x, y, 1)^T - t_r); in source s,
 *      X_s = R_s X + t_s.  The sample is valid when X_s.z > 0 and the projection (u, v) lies in [0, w_s - 1] x [0, h_s - 1];
 *      its value S is the bilinear interpolation of I_s at (u, v) with u0 = min(floor(u), w_s - 2), v0 = min(floor(v),
 *      h_s - 2) and weights u - u0, v - v0.  The device computes the same map as the plane-induced homography
 *      (u, v, 1) ~ K_s R_s R_r^T K_r^-1 (x, y, 1)^T + iota_k K_s (t_s - R_s R_r^T t_r); the two agree to rounding.
 *   4. Window: W(p) = the (2r+1)^2 reference pixels q with |q - p|_inf <= r.  p is a candidate only when W(p) lies inside the
 *      reference image.
 *   5. Per-source cost: source s is valid for (p, k) when every q in W(p) has a valid sample.  With m = (2r+1)^2, the sums
 *      A, AA of I_r(q) and I_r(q)^2, B, BB of S(q) and S(q)^2, and AB of I_r(q) S(q): var_r = m AA - A^2,
 *      var_s = m BB - B^2; the source is valid only when also var_r > m^2 min_var and var_s > m^2 min_var; then
 *      c = clamp(1 - (m AB - A B) / sqrt(var_r var_s), 0, 2).
 *   6. Aggregation: n_v = the valid sources; C_k(p) = the mean of the min(top_k, n_v) smallest c when n_v >= min_sources,
 *      else +inf.
 *   7. Winner: k* = argmin_k C_k(p), ties to the smallest k; no winner when every C_k is +inf.
 *   8. Sub-plane: C-, C0, C+ = C at k* - 1, k*, k* + 1.  When 0 < k* < n - 1, C- and C+ are finite and den = C- - 2 C0 + C+ > 0,
 *      delta = clamp((C- - C+) / (2 den), -1/2, 1/2); otherwise delta = 0.  depth = 1 / (iota_k* + delta (iota_1 - iota_0)).
 *   9. Outputs: d_depth = depth, or 0 for a non-candidate, a pixel without a winner, and C0 > max_cost; d_cost = C0, +inf
 *      without a winner; d_n_src (uint8) = n_v at k*, 0 without a winner.  *report: the candidates and the pixels with a
 *      depth.
 *  10. Determinism: a pixel's outputs depend only on its inputs; no floating-point atomics; two identical calls give
 *      identical bytes.
 * Errors: PS_ERR_ARG before any device work, with every output untouched, for: n_sets, n_refs or a CSR count < 0; NULL
 * prm, report, or (n_refs > 0) images, cams, poses, refs, ranges, src_start, src_sets (when some reference has a source) or
 * an output array; a reference or source outside [0, n_sets), a duplicate reference, a source equal to its reference;
 * src_start not running non-decreasing from 0; an image of a reference or source whose data is not device memory on
 * `device`, whose width or height is < 2r + 1 or > 65535, or whose pitch is < width; an output pointer that is not device
 * memory on `device`; a range that is not finite with 0 < d_min < d_max; a camera or pose of a reference or source that
 * ps_triangulate_tracks refuses (fx, fy finite and > 0, cx, cy finite; finite pose, max |R^T R - I| <= 1e-6, det R > 0);
 * a parameter outside its range above.  n_refs = 0 is valid: the report is zero and nothing is read.  Synchronous.
 * Workspace from the library's memory pool: 64 bytes per reference, 80 per (reference, source) and 8 per 32 x 16 tile. */
int ps_depth_maps(int device, int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs,
                  const int32_t* refs, const float* ranges, const int32_t* src_start, const int32_t* src_sets,
                  const ps_depth_params* prm, float* const* d_depth, float* const* d_cost, uint8_t* const* d_n_src,
                  ps_depth_report* report);

/* Geometric consistency between the depth maps of one call (ps_depth_maps' outputs, or any maps in its layout) and the
 * compaction of the consistent pixels into points.  images, cams, poses, refs, src_start and src_sets are as in
 * ps_depth_maps; d_depth[j] (HOST array of DEVICE pointers) is reference j's map.  In double, for each pixel p = (x, y) of
 * reference r with depth D > 0 and each source s of r that is also a reference of this call (its map D_s):
 *   1. X = R_r^T (D K_r^-1 (x, y, 1)^T - t_r), X_s = R_s X + t_s.  Needs X_s.z > 0 and pi_s(X_s) = (fx X_s.x / X_s.z + cx,
 *      fy X_s.y / X_s.z + cy) in [0, w_s - 1] x [0, h_s - 1]; q = floor(pi_s + 1/2) per coordinate; D' = D_s(q) > 0.
 *   2. X' = R_s^T (D' K_s^-1 (q, 1)^T - t_s), X'_r = R_r X' + t_r; needs X'_r.z > 0; p' = pi_r(X'_r).
 *   3. Consistent when |p' - p| <= max_reproj_error (Euclidean, pixels) and |X_s.z - D'| <= max_depth_diff D'.
 * n_consistent = the consistent sources, saturated at 255; written to d_n_consistent[j] (uint8, w x h, 0 where D <= 0).
 * Every pixel with n_consistent >= min_consistent gives one ps_dense_point (X rounded to float, ref = j, grey = I_r(x, y)),
 * compacted into d_points in (ref, y, x) order by an exclusive scan; d_points (DEVICE) holds sum over the references of
 * w h records.  *report: the pixels with D > 0 and the records written.  Deterministic: integer scan, no floating-point
 * atomics.  Errors as ps_depth_maps (its parameters aside: an image's width or height only needs to be >= 1 and <= 65535),
 * plus a filter parameter outside its range above, and a d_depth or d_n_consistent entry or d_points that is not device
 * memory on `device` (n_refs > 0); sum of w h >= 2^31.  n_refs = 0 is valid.  Synchronous; one read-back of the totals.
 * Workspace: 184 bytes per reference, 4 per (reference, source that is a reference), and 4 per pixel plus the scan's
 * partials (about 1/4096 of that). */
int ps_depth_filter(int device, int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs,
                    const int32_t* refs, const int32_t* src_start, const int32_t* src_sets, const float* const* d_depth,
                    const ps_depth_filter_params* prm, uint8_t* const* d_n_consistent, ps_dense_point* d_points,
                    ps_depth_filter_report* report);

#ifdef __cplusplus
}
#endif

#endif
