/* Global camera poses (an addition to the reference's interface): robust rotation averaging over the view graph, then
 * global positioning of the camera centres and track points, as global structure-from-motion systems do (Theia,
 * OpenMVG's global pipeline, GLOMAP).
 *
 * ps_triangulate_tracks and ps_bundle_adjust need a pose for every image.  These two entry points make those poses from
 * what the device chain already has: ps_rotation_averaging turns the relative rotations of ps_relative_pose_batch into
 * one rotation per image, and ps_global_positioning places the camera centres and the tracks' points from the unit
 * viewing rays of the tracks' observations, rotations held.  Both are IRLS loops around a weighted graph Laplacian
 * (3 unknowns per node) solved by Jacobi-preconditioned conjugate gradients on the device.  Their outputs feed
 * ps_triangulate_tracks and then ps_bundle_adjust.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_GLOBAL_H
#define POPSIFT_B200_GLOBAL_H

#include "popsift_b200_bundle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_rotation_params {    /* 40 bytes */
    int32_t loss;                      /* PS_LOSS_* (popsift_b200_bundle.h)                                          */
    int32_t max_iters;                 /* IRLS iterations, 0 .. 10000                                                */
    int32_t cg_max_iters;              /* CG iterations per IRLS iteration, 1 .. 10000                               */
    int32_t min_inliers;               /* a pair is used when n_front >= min_inliers; >= 0                           */
    double  loss_scale;                /* s, degrees; finite and > 0                                                 */
    double  step_tol;                  /* degrees; finite, >= 0                                                      */
    double  cg_tol;                    /* finite, in [0, 1)                                                          */
} ps_rotation_params;

enum {
    PS_RA_MAX_ITERS = 0,               /* max_iters IRLS iterations ran                                              */
    PS_RA_STEP_TOL = 1,                /* the largest |x_i| of an iteration was below step_tol                       */
    PS_RA_NO_PAIRS = 2                 /* no used pair in the registered component                                   */
};

typedef struct ps_rotation_report {    /* 40 bytes, HOST */
    double  initial_cost, final_cost;  /* 1/2 sum s^2 rho(|r|^2 / s^2), residuals and s in radians                   */
    int32_t iterations;                /* IRLS iterations (linear solves)                                            */
    int32_t cg_iterations;             /* summed over the iterations                                                 */
    int32_t n_pairs;                   /* used pairs of the registered component                                     */
    int32_t n_registered;              /* registered sets                                                            */
    int32_t termination;               /* PS_RA_*                                                                    */
    int32_t pad_;
} ps_rotation_report;

/* Rotation averaging.  pairs (HOST, 2 per pair: l, r, each in [0, n_sets)) and d_two_view (DEVICE, one ps_two_view per pair,
 * what ps_relative_pose_batch wrote: X_r = R_p X_l + t_p).  Rotations are world -> camera (X_cam = R_i X_world + t_i, the
 * convention of ps_rigid), so a pair says R_r = R_p R_l.  All arithmetic in double.  The float R_p of a used pair is made
 * orthonormal by a unit-quaternion round trip (k_global.h: gl_orthonormal), so that rotations chained along long paths stay
 * rotations to double precision (and pass ps_global_positioning's check).
 *   1. Used pairs: n_front >= min_inliers, every entry of R_p finite, l != r.
 *   2. Registered sets: the sets of the largest connected component of the used pairs (a set without a used pair is a
 *      component of its own); a tie goes to the component holding the smallest set id.  Only the used pairs inside it
 *      take part below; the other sets get registered = 0 and R_out = I.
 *   3. Start, on the host, once per call (this reads the n_pairs 128-byte records back once, and is sequential, O(P log P)):
 *      a maximum spanning tree of the used pairs by n_front (Kruskal, ties to the smaller pair index); the root is the
 *      smallest registered set, R = I; the other rotations follow along the tree from the root, R_r = R_p R_l when l is
 *      known, R_l = R_p^T R_r when r is known.
 *   4. IRLS on the device, the root held.  Residual of pair p: r_p = Log(R_r^T R_p R_l) (k_global.h: gl_log).  Update
 *      R_i <- R_i Exp(x_i) (Rodrigues, ps_bundle_adjust's rule), so the linearised residual is r_p + x_l - x_r.  Weights
 *      w_p = rho'(|r_p|^2 / s^2), s = loss_scale in radians.  Each iteration minimises sum w_p |r_p + x_l - x_r|^2: the
 *      weighted Laplacian system solved by CG from x = 0 with the weighted degree as the (Jacobi) preconditioner, stopped
 *      at |r| <= cg_tol |r_0| or after cg_max_iters iterations.  The loop stops after max_iters iterations, or after an
 *      iteration whose largest |x_i| is below step_tol (converted to radians).
 *   5. Outputs.  R_out (HOST, 9 per set, row-major), registered (HOST, a byte per set), pair_error (HOST, optional, a float
 *      per pair): the final |r_p| in degrees of the used pairs of the registered component, +inf for the others.
 *      *report: costs (at the start of 4 and at the end), iterations, CG iterations, counts, termination.
 *   6. Determinism: every reduction runs in a fixed order without floating-point atomics; two identical calls give
 *      identical bytes.
 * Errors: PS_ERR_ARG for n_sets or n_pairs < 0; prm, R_out, registered or report NULL; pairs NULL with n_pairs > 0, or an
 * index outside [0, n_sets); d_two_view not device memory on `device` with n_pairs > 0; a parameter outside its range
 * above.  On PS_ERR_ARG no output is written.  n_sets = 0 and n_pairs = 0 are valid (with n_sets > 0 and no pair, set 0
 * alone is registered).  Synchronous; one small read-back per iteration.
 * Workspace from the matcher's memory pool: 112 bytes per pair (its rotation, ends, weight and right-hand side, error
 * and cost partial), 8 bytes per pair end (the incidence lists) and 200 bytes per set. */
int ps_rotation_averaging(int device, int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view,
                          const ps_rotation_params* prm, double* R_out, uint8_t* registered, float* pair_error,
                          ps_rotation_report* report);

typedef struct ps_position_params {    /* 40 bytes */
    int32_t loss;                      /* PS_LOSS_*                                                                  */
    int32_t max_iters;                 /* majorise-minimise iterations after the linear start, 0 .. 10000            */
    int32_t cg_max_iters;              /* 1 .. 10000                                                                 */
    int32_t pad_;                      /* ignored                                                                    */
    double  loss_scale;                /* s; finite and > 0 (residuals are differences of unit vectors)              */
    double  function_tol;              /* finite, >= 0                                                               */
    double  cg_tol;                    /* finite, in [0, 1)                                                          */
} ps_position_params;

enum {
    PS_GP_MAX_ITERS = 0,               /* max_iters iterations ran                                                   */
    PS_GP_FUNCTION_TOL = 1,            /* an iteration decreased the cost by less than function_tol relative         */
    PS_GP_NO_OBSERVATIONS = 2          /* no used observation                                                        */
};

typedef struct ps_position_report {    /* 40 bytes, HOST */
    double  initial_cost, final_cost;  /* the reduced cost of step 2 after the linear start and at the end           */
    int32_t iterations;                /* iterations after the linear start                                          */
    int32_t cg_iterations;             /* summed over every solve, the linear start's included                       */
    int32_t n_obs;                     /* used observations                                                          */
    int32_t n_points;                  /* tracks that take part                                                      */
    int32_t n_cams;                    /* positioned sets                                                            */
    int32_t termination;               /* PS_GP_*                                                                    */
} ps_position_report;

/* Global positioning.  n_sets, n_feat, d_feat, cams, n_tracks, d_track_start, d_members and n_members are
 * ps_triangulate_tracks' arguments with the same meaning and checks; R (HOST, 9 per set, row-major world -> camera, the
 * check of ps_triangulate_tracks' poses on its rotation part) and registered (HOST, a byte per set, 0 or 1) are what
 * ps_rotation_averaging wrote.  All arithmetic in double.
 *   1. Observations: member k of set i with registered[i] = 1 is an observation of camera i and its track t; a track takes
 *      part when it has >= 2 observations, and only the observations of those tracks are used.  v_k is the member's unit
 *      world ray, ps_triangulate_tracks' step 1 (k_triangulate.h: tri_direction) under R_i.
 *   2. Cost (GLOMAP's): 1/2 sum over used observations of s^2 rho(|v_k - d_k (X_t - c_i)|^2 / s^2), c_i the camera centre
 *      and X_t the point, minimised over d_k >= 0, which gives d_k = max(0, v_k.u) / (u.u), u = X_t - c_i (d_k = 0 when
 *      u = 0).  The root, the smallest positioned set (a registered set with a used observation), holds c = 0.
 *   3. Linear start: every position 0, d = 1, w = 1, and one solve of 4.  No random start (unlike GLOMAP).
 *   4. Each later iteration is a majorise-minimise step, so the cost does not increase: d_k and w_k = rho'(.) at the
 *      current positions, then sum w_k |v_k - d_k (X_t - c_i)|^2 is minimised over the free centres and points.  That is
 *      a weighted Laplacian on the bipartite camera-point graph with edge weights w_k d_k^2 and right-hand side
 *      +-w_k d_k v_k, solved for the change of the positions by CG from 0 (the rule of ps_rotation_averaging's step 4:
 *      Jacobi preconditioner, cg_tol, cg_max_iters).  CG from the current positions never increases that quadratic, so a
 *      truncated solve keeps the guarantee.  The step x of that solve is then lengthened: the positions + 2^k x are tried
 *      for k = 1, 2, .. 20 while the cost keeps decreasing, and the last decrease is kept (the alternation between d and
 *      the positions alone creeps along one direction on short baselines; the longer steps cut the iterations needed
 *      several-fold and keep the cost from increasing).  A node without an edge of positive weight keeps its position; no proximal
 *      term.  Only the root is held: when the observations split the cameras into groups that share no track (for
 *      instance after global_poses drops pairs), each group without the root keeps a free translation and its placement
 *      relative to the root is arbitrary though reported positioned; run such groups separately.  The loop stops after max_iters iterations, or after one that decreased the cost by less than function_tol
 *      times the cost before it.
 *   5. Outputs: every position is scaled so that the RMS distance of the positioned centres from the root is 1 (not
 *      scaled when the root is the only one).  poses_out (HOST, a ps_rigid per set): (R_i, -R_i c_i) for positioned sets,
 *      (R_i, 0) for the others; positioned (HOST, a byte per set); d_X (DEVICE, optional, 3 doubles per track): the scaled
 *      points of the tracks that take part, 0 for the others.  *report: costs, iterations, CG iterations, counts,
 *      termination.
 *   6. Determinism: as ps_rotation_averaging's.
 * Errors: PS_ERR_ARG for everything ps_triangulate_tracks refuses about the sets, cameras and tracks (with R in the place
 * of the poses); prm, poses_out, positioned, report or registered NULL with n_sets > 0; a registered entry other than 0 or
 * 1; a parameter outside its range; a non-NULL d_X that is not device memory on `device` with n_tracks > 0.  A member id or
 * d_track_start out of range is found on the device and flagged before any output is written.  On PS_ERR_ARG no output is
 * written.  n_tracks = 0 is valid (NO_OBSERVATIONS, every set unpositioned).  Synchronous; one small read-back per
 * iteration.
 * Workspace from the matcher's memory pool: 84 bytes per member (its set, pixel, ray, ends, weight, right-hand side and
 * the two sort buffers), 24 bytes per track (its point) and 160 bytes per node (cameras and tracks: the CG vectors),
 * plus the scan and sort scratch (about 1 KB per 4 096 members). */
int ps_global_positioning(int device, int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                          const double* R, const uint8_t* registered, int n_tracks, const int32_t* d_track_start,
                          const int32_t* d_members, int n_members, const ps_position_params* prm, ps_rigid* poses_out,
                          uint8_t* positioned, double* d_X, ps_position_report* report);

#ifdef __cplusplus
}
#endif

#endif
