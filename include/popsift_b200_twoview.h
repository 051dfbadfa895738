/* Two-view configuration (an addition to the reference's interface): tell general, planar and panoramic pairs apart from
 * the inlier counts of their essential matrix, fundamental matrix and homography, and pose planar and panoramic pairs
 * from the homography, as COLMAP's two-view geometry does (calibrated, planar, panoramic, uncalibrated, degenerate).
 *
 * Under a pure rotation (tripod pans, panoramas, a drone yawing in hover) every E = [t]x R fits the points whatever t is,
 * so ps_relative_pose_batch returns an arbitrary t, and its cheirality choice between R and the "twisted" rotation is
 * decided by noise.  When all points lie on one plane, E is not unique either.  This entry point takes the outputs of
 * ps_verify_batch (H and F) and ps_relative_pose_batch (E) on the same rows of ps_match_correspondences and writes one
 * record and mask per pair in ps_relative_pose_batch's layout, so that the view-graph filter, rotation averaging and the
 * tracks take them unchanged: the essential pose for general pairs, the homography's pose for planar pairs, the rotation
 * alone for panoramic pairs, and no model for the others.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_TWOVIEW_H
#define POPSIFT_B200_TWOVIEW_H

#include "popsift_b200_pose.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { PS_TV_DEGENERATE = 0, PS_TV_GENERAL = 1, PS_TV_PLANAR = 2, PS_TV_PANORAMIC = 3, PS_TV_UNCALIBRATED = 4 };

typedef struct ps_two_view_config_params {  /* 32 bytes */
    int32_t min_inliers;          /* >= 0; COLMAP's default is 15                                              */
    float   threshold;            /* pixels, the pure-rotation test of step 3; finite and > 0                  */
    double  min_ef_ratio;         /* [0, 1]; COLMAP's min_E_F_inlier_ratio is 0.95                             */
    double  max_h_ratio;          /* [0, 1]; COLMAP's max_H_inlier_ratio is 0.8                                */
    double  min_rotation_ratio;   /* [0, 1]; the share of H inliers a pure rotation must explain (0.9)         */
} ps_two_view_config_params;

typedef struct ps_two_view_info {   /* 40 bytes, HOST, one per pair */
    int32_t config;                 /* PS_TV_*                                                                  */
    int32_t n_e, n_f, n_h;          /* the three models' inlier counts (step 1)                                  */
    int32_t n_rotation;             /* H-inlier rows the pure rotation R0 explains (0 unless step 3 ran)         */
    float   tri_angle;              /* median triangulation angle of the bit-1 rows, degrees; 0 if none (step 6) */
    float   normal[3];              /* PLANAR: unit plane normal in the left frame; zero otherwise               */
    int32_t pad_;
} ps_two_view_info;

/* Batched two-view configuration.  d_corr, corr_start, n_corr and cams are exactly what ps_relative_pose_batch takes
 * (DEVICE float4 rows in pixels, 16-byte aligned; HOST starts, counts and two cameras per pair, left then right); the
 * pair's calibrated rows x^ are that call's (its rule 1, the same code).  The models come from the three calls on those
 * rows: d_essential and d_essential_mask (DEVICE) from ps_relative_pose_batch; d_f_inliers (DEVICE, an int32 per pair) the
 * counts of ps_verify_batch with PS_GEOM_FUNDAMENTAL; d_homography (DEVICE, 9 floats per pair, pixels, left to right) and
 * d_h_mask (DEVICE, a byte per row) from ps_verify_batch with PS_GEOM_HOMOGRAPHY.  prm is host memory.  An "H-inlier row"
 * below is a row with a nonzero d_h_mask byte.
 *   1. Counts: n_e = d_essential[p].n_inliers, n_f = d_f_inliers[p], n_h = the number of H-inlier rows of the pair.
 *   2. Classification, in double:  calibrated = n_e >= min_inliers and n_e >= min_ef_ratio * n_f;  m = n_e when calibrated,
 *      else n_f;  planar_or_panoramic = n_h >= min_inliers and n_h > max_h_ratio * m.
 *        neither: UNCALIBRATED when n_f >= min_inliers, else DEGENERATE;
 *        calibrated and not planar_or_panoramic: GENERAL;
 *        planar_or_panoramic: step 3.
 *   3. Pure rotation.  a_i, b_i = the unit rays (x^, y^, 1) / |(x^, y^, 1)| of the left and right calibrated rows, in double.
 *      B = sum over the H-inlier rows of b_i a_i^T, per-thread partials in row order and ps_verify_batch's fixed-order block
 *      sum.  R0 = U V^T with U, V the singular vectors of B by ps_relative_pose_batch's SVD (its rule 7: det U = det V = +1,
 *      which is Kabsch's U diag(1, 1, det(U V^T)) V^T); B of rank < 2 gives n_rotation = 0.  A row passes the rotation
 *      test when, with w = R0 (x^_l, y^_l, 1) in double, w_z > 0 and (fx_r w_x / w_z + cx_r - x_r)^2 + (fy_r w_y / w_z +
 *      cy_r - y_r)^2 < threshold^2 in pixels.  n_rotation = the H-inlier rows that pass.  PANORAMIC when
 *      n_rotation >= min_rotation_ratio * n_h.
 *   4. Homography (the planar_or_panoramic pairs that are not panoramic).  H_c = K_r^-1 H K_l in double, divided by its
 *      middle singular value (the square roots of the eigenvalues of H_c^T H_c by ps_relative_pose_batch's Jacobi, sorted
 *      descending, with eigenvectors v1, v2, v3, each signed so that its first entry of largest magnitude is positive); negated when fewer than half of the H-inlier rows have
 *      (x^_r, y^_r, 1) H_c (x^_l, y^_l, 1)^T > 0.  sigma1 - sigma3 <= 1e-9 sigma2: no parallax, PANORAMIC.  Otherwise the
 *      four (R, t, n) with H_c = R + t n^T, |n| = 1, by the SVD method of Faugeras-Lustman / Ma-Soatto-Kosecka-Sastry (An
 *      Invitation to 3-D Vision, 5.3), with s1 >= s2 >= s3 the singular values of the normalised H_c:
 *      u+- = (sqrt(s2^2 - s3^2) v1 +- sqrt(s1^2 - s2^2) v3) / sqrt(s1^2 - s3^2),
 *      U = [v2, u, v2 x u], W = [H_c v2, H_c u, H_c v2 x H_c u], R = W U^T, n = v2 x u, t = (H_c - R) n; in order
 *      (u+, n), (u-, n), (u+, -n, -t), (u-, -n, -t).  The candidates with n_z > 0 are kept in that order (two, unless an n_z
 *      is exactly 0); each is scored by the H-inlier rows in front under ps_relative_pose_batch's pose_front with
 *      (R, t / |t|); the most rows win, ties to the lower index.  No candidate left, or a homography that is zero or not
 *      finite: the pair is classified by step 2 as if planar_or_panoramic were false.  Otherwise PLANAR.
 *   5. Outputs.  d_out (DEVICE, a ps_two_view per pair), d_out_mask (DEVICE, a byte per row: bit 0 inlier, bit 1 bit 0
 *      and in front; the only values are 0, 1 and 3, a valid d_inlier_mask for ps_tracks_from_matches), d_points
 *      (DEVICE, optional, a float4 per row: (X, Y, Z, 1) in the left frame for rows with bit 1, zero otherwise).
 *        GENERAL: d_out[p] is d_essential[p] byte for byte and the mask is d_essential_mask; the points are
 *          ps_relative_pose_batch's rule 8 under its output R and t (byte for byte what it writes to d_points).
 *        PLANAR: R and t = the chosen candidate's R and t / |t| rounded to float32, E = [t]x R / sqrt(2) and F = K_r^-T E
 *          K_l^-1 as in ps_relative_pose_batch's rule 8; bit 0 = the H mask, bit 1 = bit 0 and pose_front under the output
 *          R and t; n_inliers, n_front count the bits; points as in rule 8.  normal = n rounded to float32.
 *        PANORAMIC: R = R0 rounded to float32, t = 0, E = F = 0 (a zero model gives no guided rows);
 *          bit 0 = the H mask, bit 1 = bit 0 and the rotation test of step 3; n_inliers = n_h, n_front = n_rotation;
 *          points zero.
 *        UNCALIBRATED, DEGENERATE: the record, the mask and the points are zero, ps_relative_pose_batch's "no model"
 *          record, which rotation averaging, the view-graph filter and the tracks ignore.
 *   6. tri_angle (GENERAL and PLANAR): for each bit-1 row, X its point in double (before rounding) and c = -R^T t the right
 *      centre under the output R and t, the angle between X and X - c, atan2(|X x (X - c)|, X . (X - c)) in degrees,
 *      rounded to float32; tri_angle is the lower median of those angles (rank floor((k - 1) / 2) of k, exact: a radix
 *      select on the float bit patterns).  Zero when k = 0 and for every other configuration.  It is COLMAP's
 *      TwoViewGeometry::tri_angle: small values flag pairs with little baseline.
 *   7. Determinism: results depend only on the inputs; fixed-order double sums and integer counts only, so two identical
 *      calls give identical bytes.
 * Errors: PS_ERR_ARG, with no output written, for everything ps_relative_pose_batch refuses about rows and cameras
 * (negative counts or starts, NULL corr_start / n_corr / cams with n_pairs > 0, an fx or fy that is not finite and > 0, a
 * cx or cy that is not finite, d_corr not 16-byte aligned); prm or info NULL; min_inliers < 0, a threshold that is not
 * finite and > 0, a ratio outside [0, 1]; a device pointer (d_corr, the masks when some pair has rows; d_essential,
 * d_f_inliers, d_homography, d_out; a non-NULL d_points) that is not device memory on `device`; an output range that
 * overlaps an input range or another output (host range check on the sizes above).  n_pairs = 0 is valid.  Synchronous;
 * one read-back of info.  Workspace from the library's memory pool: 128 bytes per pair (its rows, cameras and info) and 4
 * per row (the angle bits). */
int ps_two_view_config_batch(int device, int n_pairs, const float* d_corr, const int32_t* corr_start, const int32_t* n_corr,
                             const ps_camera* cams, const ps_two_view* d_essential, const uint8_t* d_essential_mask,
                             const int32_t* d_f_inliers, const float* d_homography, const uint8_t* d_h_mask,
                             const ps_two_view_config_params* prm, ps_two_view* d_out, uint8_t* d_out_mask, float* d_points,
                             ps_two_view_info* info);

#ifdef __cplusplus
}
#endif

#endif
