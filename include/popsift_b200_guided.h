/* Guided matching (an addition to the reference's interface): 2-NN matching of many pairs of descriptor sets, where the
 * candidates of a left descriptor are only the right descriptors whose keypoints agree with the pair's two-view model.
 *
 * The ratio test of ps_match_batch runs over the whole right image, so it rejects a correct match whenever the second-
 * nearest descriptor is a repeat of the same structure elsewhere (windows, tiles, texture).  Geometric verification
 * (ps_verify_batch) finds the model that rules those repeats out; guided matching then matches every pair again with
 * only the right descriptors that fit the model as candidates (COLMAP's guided_matching, SiftGPU's GetGuidedSiftMatch).
 * The chain extract -> ps_match_batch -> ps_match_correspondences -> ps_verify_batch -> ps_match_guided_batch ->
 * ps_match_correspondences never leaves the device.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_GUIDED_H
#define POPSIFT_B200_GUIDED_H

#include "popsift_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Inputs.  Sets, pair list, flags and output layout are those of ps_match_batch (float descriptors) and ps_match_u8_batch
 * (8-bit descriptors, 16-byte aligned).  d_feat[i] / d_rev[i] are the Feature records and the descriptor -> feature
 * reverse map of ps_download_dev (DEVICE, on `device`), as ps_match_correspondences takes them; d_sets, d_feat, d_rev,
 * n_desc and pairs are host arrays.  d_models (DEVICE) holds 9 floats per pair, row-major, mapping left to right in pixels:
 * exactly the d_models output of ps_verify_batch.  `model` (PS_GEOM_HOMOGRAPHY / PS_GEOM_FUNDAMENTAL) applies to every pair;
 * `threshold` t is in pixels.
 *
 * Eligibility.  Right descriptor j is eligible for left descriptor i of pair p when the pixel points
 * x_l = feat_l[rev_l[i]].(xpos, ypos) and x_r = (X, Y) = feat_r[rev_r[j]].(xpos, ypos) pass ps_verify_batch's inlier test
 * under model p, evaluated in pixel coordinates in float32, each step rounded once (fma = one rounding):
 *     t2 = t * t
 *     homography   u = fma(m0, x, fma(m1, y, m2)),  v = fma(m3, x, fma(m4, y, m5)),  w = fma(m6, x, fma(m7, y, m8))
 *                  du = fma(-X, w, u),  dv = fma(-Y, w, v)
 *                  eligible when  fma(du, du, dv * dv) < t2 * (w * w)          [(u - X w)^2 + (v - Y w)^2 < t^2 w^2]
 *     fundamental  a0, a1, a2 = F x_l as u, v, w above;  ra = fma(a0, a0, a1 * a1)
 *                  b0 = fma(m0, X, fma(m3, Y, m6)),  b1 = fma(m1, X, fma(m4, Y, m7)),  cb = fma(b0, b0, b1 * b1)
 *                  e = fma(X, a0, fma(Y, a1, a2))
 *                  eligible when  e * e < t2 * (ra + cb)                      [e^2 < t^2 (a0^2 + a1^2 + b0^2 + b1^2)]
 *   The comparison is strict, so a zero model (what ps_verify_batch writes for a pair where it found none) makes nothing
 *   eligible, and so does a NaN anywhere: such a pair yields rows (0, 0, 0) and no correspondences.
 *
 * Rows.  Row i of pair p is what ps_match_batch(..., PS_MATCH_EXACT) gives on the right set restricted to the eligible
 * descriptors, with indices mapped back to the full right set: the strict-< scan in index order and accept =
 * best / second < 0.8f.  No eligible descriptor gives (0, 0, 0); exactly one, j, gives (j, 0, 1).  Empty sets, self pairs
 * and pairs in several groups follow ps_match_batch.  The float tensor path carries ps_match_batch's near-tie caveat; the
 * u8 rows are exact, and equal the float PS_MATCH_EXACT guided rows on float32 copies of the same sets.
 *
 * flags.  PS_MATCH_EXACT runs a CUDA-core guided kernel pair by pair (the in-library reference); PS_MATCH_AUTO /
 * PS_MATCH_TENSOR run the batched tensor-core path (the matcher's kernels with the test fused into their epilogue).
 *
 * Returns when the result is complete.  PS_ERR_ARG for what ps_match_batch / ps_match_u8_batch / ps_match_correspondences
 * refuse (negative counts, a set index out of range, a null pointer with a count > 0, set, Feature or reverse-map arrays
 * that are not device memory on `device`, u8 sets not 16-byte aligned), and for an unknown model, a threshold that is not
 * finite and > 0, or d_models that is not device memory on `device` when some pair has rows and a non-empty right set.
 * When no pair has both, d_models is not read and may be NULL.  n_pairs = 0 is valid. */
int ps_match_guided_batch(int device, int n_sets, const ps_descriptor* const* d_sets, const ps_feature* const* d_feat,
                          const int32_t* const* d_rev, const int32_t* n_desc, int n_pairs, const int32_t* pairs,
                          const float* d_models, int model, float threshold, int32_t* d_out, int flags);
int ps_match_u8_guided_batch(int device, int n_sets, const uint8_t* const* d_sets, const ps_feature* const* d_feat,
                             const int32_t* const* d_rev, const int32_t* n_desc, int n_pairs, const int32_t* pairs,
                             const float* d_models, int model, float threshold, int32_t* d_out, int flags);

#ifdef __cplusplus
}
#endif

#endif
