/* Bundle adjustment (an addition to the reference's interface): Levenberg-Marquardt refinement of camera poses and track
 * points on the device, with the Schur complement onto the cameras solved by preconditioned conjugate gradients.
 *
 * ps_triangulate_tracks gives one point per track from poses that are only estimates (relative-pose chaining, GNSS / SLAM
 * priors, a perturbed rig).  This entry point makes poses and points consistent with the observations, as COLMAP's and
 * Ceres' bundle adjusters do, on the tracks, Feature records, points and masks where they already are: it takes exactly
 * what ps_triangulate_tracks takes and writes, so its outputs feed this call without a host copy.  Intrinsics are held.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_BUNDLE_H
#define POPSIFT_B200_BUNDLE_H

#include "popsift_b200_triangulate.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
    PS_LOSS_SQUARED = 0,               /* rho(z) = z                                                                 */
    PS_LOSS_HUBER = 1,                 /* rho(z) = z for z <= 1, else 2 sqrt(z) - 1                                  */
    PS_LOSS_CAUCHY = 2                 /* rho(z) = ln(1 + z)                                                         */
};

typedef struct ps_bundle_params {      /* 56 bytes */
    int32_t loss;                      /* PS_LOSS_*                                                                  */
    int32_t max_iters;                 /* LM iterations, 0 .. 10000                                                  */
    int32_t cg_max_iters;              /* CG iterations per LM iteration, 1 .. 10000                                 */
    int32_t scale_set;                 /* -1, or the set one of whose translation components is held                 */
    int32_t scale_axis;                /* 0 .. 2: that component                                                     */
    int32_t pad_;                      /* ignored                                                                    */
    double  loss_scale;                /* s, pixels; finite and > 0                                                  */
    double  function_tol;              /* finite, >= 0                                                               */
    double  cg_tol;                    /* finite, in [0, 1)                                                          */
    double  initial_lambda;            /* finite, in (0, 1e32]                                                       */
} ps_bundle_params;

enum {
    PS_BA_MAX_ITERS = 0,               /* max_iters LM iterations ran                                                */
    PS_BA_FUNCTION_TOL = 1,            /* an accepted step decreased the cost by less than function_tol relative     */
    PS_BA_LAMBDA = 2,                  /* lambda > 1e32                                                              */
    PS_BA_NO_OBSERVATIONS = 3,         /* no used observation                                                        */
    PS_BA_NONFINITE_START = 4          /* the initial cost is not finite                                             */
};

typedef struct ps_bundle_report {      /* 48 bytes, HOST */
    double  initial_cost, final_cost;
    int32_t iterations;                /* LM iterations (solves), accepted or not                                    */
    int32_t accepted;                  /* accepted steps                                                             */
    int32_t cg_iterations;             /* CG iterations summed over the LM iterations                                */
    int32_t termination;               /* PS_BA_*                                                                    */
    int32_t n_obs;                     /* used observations                                                          */
    int32_t n_points;                  /* tracks with a used observation                                             */
    int32_t n_free_cams;               /* sets not fixed with a used observation                                     */
    int32_t pad_;
} ps_bundle_report;

/* Refine the poses of the free sets and the points of the OK tracks.  n_sets, n_feat, d_feat, cams, n_tracks,
 * d_track_start, d_members and n_members are ps_triangulate_tracks' arguments with the same meaning and rules (member k of
 * set i observes (x, y) = (d_feat[i][f].xpos, .ypos), the pinhole cams[i] is held fixed); poses_in (HOST) one ps_rigid
 * per set; d_points (DEVICE, n_tracks records, in/out) and d_obs_mask (DEVICE, n_members bytes, in) as
 * ps_triangulate_tracks wrote them; fixed (HOST, n_sets bytes, 0 or 1): 1 holds that set's pose.
 * All arithmetic is in double; fx, fy, cx, cy, x and y are converted exactly from float.
 *   1. Observations: member k of track t is used when d_points[t].status == PS_TRI_OK and d_obs_mask[k] != 0; nothing
 *      else enters the cost.  The points are X_t = d_points[t].X of the tracks with a used observation.
 *   2. Residual (tri_residual of ps_triangulate_tracks, step 4): X_c = R X + t, iz = 1 / z,
 *      e = (fx (X_c[0] iz) + cx - x, fy (X_c[1] iz) + cy - y); a used observation with z <= 0 makes the cost +inf.
 *   3. Cost: 1/2 sum over used observations of s^2 rho(|e|^2 / s^2), s = loss_scale (the loss applies to the squared norm
 *      of each 2-vector residual, as in Ceres and COLMAP).
 *   4. Parameters: a free set's pose R <- Exp(w) R (Rodrigues: theta2 = w.w, A = sin(theta) / theta, B = (1 - cos(theta))
 *      / theta2, or 1 - theta2 / 6 and 1 / 2 - theta2 / 24 when theta2 < 1e-16; Exp(w) = I + A [w]x + B (w w^T - theta2 I)),
 *      t <- t + dt; a point X <- X + dX.  Jacobians at 0: with a_r = d e_r / d X_c and v = X_c - t, d e_r / dw = v x a_r,
 *      d e_r / d dt = a_r, d e / dX as tri_residual gives it.
 *   5. Gauge: at least one set is fixed.  When scale_set >= 0 and that set is not fixed, component scale_axis of its t is
 *      held (COLMAP's convention for the second image).  A free set without a used observation keeps its pose, and only
 *      the free sets with a used observation count as free cameras.
 *   6. Levenberg-Marquardt over the free parameters: weights w = rho'(|e|^2 / s^2) at the current parameters (IRLS, no
 *      second-order loss term), H = sum w J^T J, g = sum w J^T e.  The step solves (H + lambda D) d = -g, D = diag(H) with
 *      each entry clamped to [1e-6, 1e32]; lambda starts at initial_lambda, nu = 2.  pred = -(g.d + 1/2 d^T H d).  The
 *      step is accepted when the new cost is finite and lower: then rho = (old - new) / pred, lambda *= max(1/3,
 *      1 - (2 rho - 1)^3) (1/3 when pred <= 0 or rho is not finite), nu = 2; otherwise lambda *= nu, nu *= 2.  Stops
 *      after max_iters iterations (accepted or not), on an accepted step with (old - new) < function_tol old, or when
 *      lambda > 1e32.
 *   7. Linear solve: the Schur complement onto the free cameras.  The point blocks V_j + lambda D_j (3 x 3) are inverted
 *      directly (a block whose determinant is not finite and > 0 leaves its point unchanged).  S = U - W V^-1 W^T is
 *      never formed: preconditioned CG from x = 0 applies it as two passes over the observations (track-major, then
 *      camera-major).  The preconditioner is block-Jacobi: the exact 6 x 6 diagonal blocks of S by Cholesky (a block
 *      whose factorisation fails is replaced by the identity); a held translation component is removed from its block.
 *      CG stops at |r| <= cg_tol |r_0| or after cg_max_iters iterations; the points follow by back-substitution.
 *   8. Outputs.  poses_out (HOST, n_sets, may alias poses_in): the final poses; they pass ps_triangulate_tracks' pose
 *      check.  d_points: for every OK track with a used observation, X is the final point and error / angle are
 *      recomputed by ps_triangulate_tracks' rules (step 7 there) over the used observations; n_inliers and status are
 *      not changed; every other record keeps its bytes.  d_obs_error (DEVICE, optional): the final pixel error sqrt(e2)
 *      as float of every member of an OK track (used or not, +inf when z <= 0), +inf for the members of other tracks.
 *      *report: costs, iterations, accepted steps, CG iterations, termination and counts.
 *   9. With no used observation (NO_OBSERVATIONS) or a non-finite initial cost (NONFINITE_START) the call returns PS_OK,
 *      poses_out = poses_in, d_points keeps its bytes; d_obs_error is written.
 *  10. Determinism: every reduction (costs, gradients, the U and V blocks, CG's dot products) runs in a fixed order,
 *      without floating-point atomics; two identical calls give identical bytes.
 * Errors: PS_ERR_ARG for everything ps_triangulate_tracks refuses (with d_points and d_obs_mask in the place of its
 * outputs); poses_out, fixed, prm or report NULL; a fixed entry other than 0 or 1, or no fixed set; scale_set outside
 * [-1, n_sets) or scale_axis outside [0, 2]; a parameter outside its range above.  A member id or d_track_start out of
 * range is found on the device and flagged before any output is written.  On PS_ERR_ARG no output is written.
 * Synchronous: returns when the result is complete; one small read-back per LM iteration.
 * Workspace from the matcher's memory pool: 16 bytes per member for its set, pixel and used-flag scan, 180 bytes per used
 * observation (the stored weighted Jacobians and residual, its member, track and set, the two sort buffers), sized for
 * every member since the used count is known only on the device; 216 bytes per track; 1 232 bytes per set; and the
 * scan's partial sums and the radix sort's histograms (about 1 KB per 4 096 members). */
int ps_bundle_adjust(int device, int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                     const ps_rigid* poses_in, int n_tracks, const int32_t* d_track_start, const int32_t* d_members, int n_members,
                     ps_track_point* d_points, const uint8_t* d_obs_mask, const uint8_t* fixed, const ps_bundle_params* prm,
                     ps_rigid* poses_out, float* d_obs_error, ps_bundle_report* report);

#ifdef __cplusplus
}
#endif

#endif
