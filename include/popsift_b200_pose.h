/* Calibrated two-view geometry (an addition to the reference's interface): batched five-point RANSAC essential matrices,
 * the relative pose (R, t) of each pair and its triangulated inliers.
 *
 * ps_verify_batch fits a homography or an uncalibrated fundamental matrix in pixels.  A structure-from-motion system that
 * knows its intrinsics estimates the essential matrix instead, decomposes it into a relative pose and triangulates the
 * inliers to choose among its four decompositions (COLMAP's calibrated two-view geometry; OpenCV's findEssentialMat +
 * recoverPose).  This entry point does that for many pairs in one call on the device, on the rows of
 * ps_match_correspondences, so the chain extract -> ps_match_batch -> ps_match_correspondences -> pose never leaves it.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_POSE_H
#define POPSIFT_B200_POSE_H

#include "popsift_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_camera { float fx, fy, cx, cy; } ps_camera;           /* 16 bytes: pinhole intrinsics in pixels */

typedef struct ps_pose_params {      /* 24 bytes */
    int32_t  n_samples;   /* minimal samples per pair, 1 .. 65536 (fixed; no early exit)        */
    float    threshold;   /* pixels; finite and > 0                                             */
    int32_t  refine;      /* 1: one least-squares refit on the winner's inliers; 0: none        */
    int32_t  pad_;        /* ignored                                                            */
    uint64_t seed;
} ps_pose_params;

typedef struct ps_two_view {         /* 128 bytes, one per pair, DEVICE */
    float   E[9];         /* calibrated coordinates, row-major, x_r^T E x_l = 0: [t]x R / sqrt(2) */
    float   F[9];         /* pixels: K_r^-T E K_l^-1, scaled like ps_verify_batch's F            */
    float   R[9];         /* row-major; X_r = R X_l + t                                          */
    float   t[3];         /* unit length                                                         */
    int32_t n_inliers;    /* rows with mask bit 0                                                */
    int32_t n_front;      /* rows with mask bit 1                                                */
} ps_two_view;

/* Batched calibrated RANSAC.  d_corr, corr_start and n_corr are exactly what ps_verify_batch takes (pair p's rows are
 * corr_start[p] .. corr_start[p] + n_corr[p] - 1 of d_corr: DEVICE float4 x_l, y_l, x_r, y_r in pixels, 16-byte aligned),
 * so the rows of ps_match_correspondences feed it unchanged.  cams (HOST) holds two cameras per pair, left then right;
 * prm is host memory.  Points must already be undistorted: the pinhole model only.
 *   1. Calibrated points: x^ = (x - cx) / fx, y^ = (y - cy) / fy in double, rounded once to float32 (a float4 row per
 *      correspondence).  f = (fx_l + fy_l + fx_r + fy_r) / 4 in double; the squared threshold is t2 = (float)((threshold /
 *      f)^2).
 *   2. Inlier test: ps_verify_batch's fundamental test (the Sampson distance, same float32 expression, same device
 *      function) on the calibrated rows against t2.
 *   3. Samples: ps_verify_batch's hash with m = 5, key (seed, p, s); a sample without 5 distinct indices after 64 draws is
 *      invalid, and so is every sample of a pair with n < 5.
 *   4. Hypotheses: h = 10 s + j.  The five-point method in double, one lane per sample:
 *        the 5 x 9 system of x_r^T E x_l = 0 (row (x_r x_l, x_r y_l, x_r, y_r x_l, y_r y_l, y_r, x_l, y_l, 1)) by Gauss-Jordan
 *          elimination with partial pivoting in column order; a column whose largest remaining entry is <= 1e-10 times the
 *          largest entry of the system is free; anything but four free columns gives no solution.  The null vectors of the
 *          free columns in order (that column 1, the other free columns 0), orthonormalised by modified Gram-Schmidt in that
 *          order, are X, Y, Z, W, and E = x X + y Y + z Z + W;
 *        the ten cubics det E = 0 and 2 E E^T E - tr(E E^T) E = 0 in 20 monomials, ordered x^3, y^3, x^2y, xy^2, x^2z, x^2,
 *          y^2z, y^2, xyz, xy | xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1;
 *        Gauss-Jordan elimination of the 10 x 20 matrix with partial pivoting on the first ten columns; a pivot <= 1e-12
 *          times the largest entry of the matrix gives no solution;
 *        (row x^2z) - z (row x^2), (row y^2z) - z (row y^2), (row xyz) - z (row xy) are linear in (x, y, 1) with
 *          coefficients in z of degree 3, 3, 4; the determinant of that 3 x 3 is a polynomial of degree 10 in z;
 *        its real roots, isolated by the derivative chain (the roots of p^(k+1) bound the intervals on which p^(k) is
 *          monotone, from Fujiwara's bound of p inwards) and polished by Newton steps kept inside each bracket, bisection
 *          where a step would leave it or not halve the step before.  A root of even multiplicity is not found;
 *        at each root, (x, y, 1) is the largest of the three row cross products of the 3 x 3.
 *      A root whose x, y or E is not finite, or whose E is zero, is skipped and the solutions are numbered without it: slot
 *      j holds the j-th remaining solution in ascending z, and the slots after the last one are invalid (count -1).  A hypothesis is stored as float32 E in calibrated coordinates with
 *      Frobenius norm 1 and its first entry of largest magnitude positive.
 *   5. Selection: the most inliers wins, ties to the smallest h; invalid hypotheses never win.
 *   6. Refit (refine = 1 and at least 8 inliers): the 8-point normal matrix of the winner's calibrated inlier rows
 *      (ps_verify_batch's, double, fixed order), its smallest eigenvector by the same Jacobi, projected onto the essential
 *      matrices as U diag(1, 1, 0) V^T and scaled as in 4; kept when its inlier count is >= the winner's.  Not iterated.
 *   7. Pose: the SVD of the selected E in double, U and V with det +1 (v1, v2 the eigenvectors of E^T E of the two largest
 *      eigenvalues by Jacobi, v3 = v1 x v2, u1 = E v1 / |E v1|, u2 the unit part of E v2 orthogonal to u1, u3 = u1 x u2).
 *      With W = [[0,-1,0],[1,0,0],[0,0,1]] the candidates are, in order, (U W V^T, +u3), (U W V^T, -u3), (U W^T V^T, +u3),
 *      (U W^T V^T, -u3).  For each candidate and each row that passes the inlier test under the selected E, in double:
 *      a = R (x^_l, y^_l, 1), b = (x^_r, y^_r, 1), (d_l, d_r) minimising |d_l a + t - d_r b|^2 by the 2 x 2 normal equations;
 *      the row is in front when det = (a.a)(b.b) - (a.b)^2 > 1e-12 (a.a)(b.b), d_l > 0 and d_r > 0.  The candidate with the
 *      most rows in front wins, ties to the lower index.
 *   8. Output: R and t are the winning candidate rounded to float32; E = [t]x R / sqrt(2) computed in double from those
 *      float32 R and t, so E, R and t agree by construction; F = K_r^-T E K_l^-1 in double with Frobenius norm 1 and its
 *      first entry of largest magnitude positive (a valid model row for ps_match_guided_batch with PS_GEOM_FUNDAMENTAL).
 *      d_inlier_mask (DEVICE, one byte per d_corr row): bit 0 is the inlier test under the output E, bit 1 is bit 0 and in
 *      front under the output R and t by the rule of 7; the only values are 0, 1 and 3, so the mask is a valid
 *      d_inlier_mask for ps_tracks_from_matches.  n_inliers and n_front count the two bits.
 *      d_points (DEVICE, optional): a float4 per d_corr row, (X, Y, Z, 1) in the left camera frame with unit baseline for
 *      rows with bit 1, zero otherwise; the point is the midpoint (d_l x^_l + R^T (d_r b - t)) / 2 of the two rays.
 *      n < 5 or no valid hypothesis: the pair's ps_two_view, mask and points are zero -- not an error.
 *   9. Taps (tests): ps_verify_taps with pair p's block at hypothesis p * 10 * n_samples: every hypothesis's inlier count
 *      (-1 invalid) and its calibrated E scaled as in 4 (zero when invalid).  Unlike ps_verify_batch's taps, these models are
 *      not in pixels.
 *  10. Determinism: results depend only on (seed, p, the pair's rows, its cameras, prm); two identical calls give identical
 *      bytes.
 * Degenerate scenes (pure rotation, all points on one plane) have no unique E; the result is then one of the fitting
 * essential matrices and the caller decides (for instance by comparing with ps_verify_batch's homography inliers).
 * Returns when the result is complete.  PS_ERR_ARG for what ps_verify_batch refuses other than the model (n_samples
 * outside [1, 65536], a threshold that is not finite and > 0, refine not 0 / 1, negative counts or starts, a null pointer
 * where a count is > 0, a pointer that is not device memory on `device`); cams == NULL with n_pairs > 0; an fx or fy that
 * is not finite and > 0, or a cx or cy that is not finite; d_out not device memory on `device`; a non-NULL d_points that
 * is not device memory on `device`.  n_pairs = 0 is valid.  Workspace: 44 bytes per hypothesis and 16 per row, from the
 * matcher's memory pool. */
int ps_relative_pose_batch(int device, int n_pairs, const float* d_corr, const int32_t* corr_start, const int32_t* n_corr,
                           const ps_camera* cams, const ps_pose_params* prm, ps_two_view* d_out, uint8_t* d_inlier_mask,
                           float* d_points, const ps_verify_taps* taps);

#ifdef __cplusplus
}
#endif

#endif
