/* Multi-view triangulation (an addition to the reference's interface): one robust 3-D point per feature track from known
 * camera poses.
 *
 * ps_tracks_from_edges / ps_tracks_from_matches give tracks: one physical point seen as at most one feature per image.  A
 * caller with camera poses (a calibrated rig, GNSS / INS or SLAM poses, an earlier reconstruction to re-triangulate) wants
 * a point per track: COLMAP's point_triangulator, AliceVision's triangulation node.  This entry point does that for every
 * track in one call on the device, on the tracks and Feature records where they already are: a small RANSAC over pairs of
 * each track's observations, then a Gauss-Newton refinement of the winner.  The result is what a bundle adjuster takes.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_TRIANGULATE_H
#define POPSIFT_B200_TRIANGULATE_H

#include "popsift_b200_pose.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_rigid {              /* 96 bytes: world -> camera, X_cam = R X_world + t (ps_two_view's convention) */
    double R[9];                       /* row-major; used as given, not re-orthonormalised                          */
    double t[3];
} ps_rigid;

typedef struct ps_triangulate_params { /* 32 bytes */
    float    max_error;                /* pixels; finite and > 0                                                   */
    float    min_angle;                /* degrees, in [0, 90)                                                      */
    int32_t  min_views;                /* >= 2                                                                     */
    int32_t  n_samples;                /* hypotheses per track when sampled, 1 .. 65536                            */
    int32_t  refine_iters;             /* Gauss-Newton steps, 0 .. 32                                              */
    int32_t  pad_;                     /* ignored                                                                  */
    uint64_t seed;
} ps_triangulate_params;

enum {
    PS_TRI_OK = 0,                     /* n_inliers >= min_views and the triangulation angle >= min_angle          */
    PS_TRI_TOO_FEW_OBS = 1,            /* the track has fewer than min_views members: nothing was computed         */
    PS_TRI_NO_HYPOTHESIS = 2,          /* no valid hypothesis                                                      */
    PS_TRI_TOO_FEW_INLIERS = 3,        /* n_inliers < min_views                                                    */
    PS_TRI_SMALL_ANGLE = 4             /* enough inliers, but the triangulation angle < min_angle                  */
};
#define PS_TRI_NUM_STATUS 5

typedef struct ps_track_point {        /* 40 bytes, one per track, DEVICE */
    double  X[3];                      /* world coordinates                                                        */
    float   error;                     /* mean pixel reprojection error over the inliers                           */
    float   angle;                     /* triangulation angle, degrees                                             */
    int32_t n_inliers;
    int32_t status;                    /* PS_TRI_*                                                                 */
} ps_track_point;

typedef struct ps_triangulate_counts { /* 24 bytes, HOST */
    int32_t n_status[PS_TRI_NUM_STATUS]; /* tracks per status                                                      */
    int32_t n_inlier_obs;              /* observations with d_obs_mask = 1                                         */
} ps_triangulate_counts;

/* Triangulate every track.  Set i has n_feat[i] Feature records at d_feat[i] (DEVICE; n_feat and d_feat are host arrays),
 * camera cams[i] and pose poses[i] (HOST).  d_track_start (n_tracks + 1 entries) and d_members (n_members global ids
 * off[i] + f, off[i] = sum_{j<i} n_feat[j]) are DEVICE arrays exactly as ps_tracks_from_edges / ps_tracks_from_matches
 * write them: track t's members are d_members[d_track_start[t] .. d_track_start[t + 1] - 1], L = their number.  Member
 * k's observation is (x, y) = (d_feat[i][f].xpos, .ypos) in undistorted pixels: the pinhole model only, and the same
 * coordinates ps_match_correspondences hands to ps_relative_pose_batch, so cams means the same in both calls.
 * All arithmetic below is in double; fx, fy, cx, cy, x and y are converted exactly from float.
 *   1. Rays: member k of set i has the camera centre C = -R^T t and the unit direction d = u / |u|, u = R^T ((x - cx) / fx,
 *      (y - cy) / fy, 1), each component divided by |u| = sqrt(u.u).
 *   2. Hypotheses: pairs (a, b), a < b, of the track's member positions.  When L (L - 1) / 2 <= n_samples every pair is a
 *      hypothesis and h is its rank in lexicographic order; otherwise there are n_samples hypotheses, h = s, and sample s
 *      draws two distinct positions by ps_verify_batch's hash with m = 2 and key (seed, t, s), a the smaller and b the
 *      larger (a sample without two distinct positions after 64 draws is invalid).
 *   3. Hypothesis point: (s_a, s_b) minimising |s_a d_a + (C_a - C_b) - s_b d_b|^2 by the 2 x 2 normal equations
 *      (ps_relative_pose_batch's rule, step 7 of popsift_b200_pose.h), X = ((C_a + s_a d_a) + (C_b + s_b d_b)) / 2.  Valid
 *      when det = (d_a.d_a)(d_b.d_b) - (d_a.d_b)^2 > 1e-12 (d_a.d_a)(d_b.d_b), s_a > 0, s_b > 0 and d_a.d_b <= cos(min_angle)
 *      (the cosine computed once on the host).
 *   4. Inlier test of member k under X: X_c = R X + t; z = X_c[2] > 0; iz = 1 / z; e_x = fx (X_c[0] iz) + cx - x,
 *      e_y = fy (X_c[1] iz) + cy - y; an inlier when e2 = e_x^2 + e_y^2 <= max_error^2 (squared in double from the float).
 *   5. Selection: the most inliers wins, ties to the smallest h; invalid hypotheses never win.
 *   6. Refinement: Gauss-Newton on the sum of e2 over the winner's inliers (a fixed set), at most refine_iters steps: the
 *      3 x 3 normal equations J^T J dX = -J^T e solved by Cramer's rule; a step is kept only when the sum decreases (a
 *      member of the set with z <= 0 makes the sum +inf); the first step that is not kept, or a determinant that is not
 *      finite and > 0, ends it.  Then every member is tested under the refined X; the refined X is kept when it has at least
 *      as many inliers as the winner, otherwise the hypothesis point is.  Not iterated further.
 *   7. Outputs under the final X: d_obs_mask (DEVICE, one byte per member) is the inlier test; d_obs_error (DEVICE,
 *      optional) is sqrt(e2) rounded to float, +inf when z <= 0; n_inliers counts the mask; error is the mean of sqrt(e2)
 *      over the inliers; angle is the largest angle at X between C_a - X and C_b - X over pairs of inliers (COLMAP's
 *      triangulation angle; the cosines of unit vectors compared, acos of the smallest in degrees; 0 with fewer than two
 *      inliers).  Status: TOO_FEW_INLIERS when n_inliers < min_views, else SMALL_ANGLE when the smallest cosine is >
 *      cos(min_angle), else OK.  These are written whatever the status.  A track with L < min_views (TOO_FEW_OBS) or
 *      without a winner (NO_HYPOTHESIS) gets X = 0, error = angle = 0, n_inliers = 0, mask 0 and error +inf.
 *      *counts: the tracks per status and the inlier observations.
 *   8. Determinism: a track's results depend only on (seed, t, its observations, their cameras and poses, prm); two
 *      identical calls give identical bytes.
 * Errors: PS_ERR_ARG for n_sets, n_tracks or n_members < 0; prm or counts NULL; a parameter outside its range above; a null
 * n_feat, d_feat, cams or poses with n_sets > 0; a negative n_feat or sum n_feat >= 2^31; a non-empty set whose records are
 * not device memory on `device`; an fx or fy that is not finite and > 0, a cx or cy that is not finite; a pose with an
 * entry that is not finite, max |R^T R - I| > 1e-6 or det R <= 0; d_track_start or d_points (n_tracks > 0), d_members or
 * d_obs_mask (n_members > 0), or a non-NULL d_obs_error that is not device memory on `device`.  A member id outside
 * [0, N), or a d_track_start that does not run non-decreasing from 0 to n_members, is found on the device: a flag is read
 * back before any output is written, and the call returns PS_ERR_ARG with the outputs untouched.  *counts is written only
 * when the call returns PS_OK.  n_tracks = 0 is valid:
 * the counts are zero and nothing is read.  Returns when the result is complete.
 * Workspace from the matcher's memory pool: 40 bytes per member and 164 bytes per set. */
int ps_triangulate_tracks(int device, int n_sets, const int32_t* n_feat, const ps_feature* const* d_feat, const ps_camera* cams,
                          const ps_rigid* poses, int n_tracks, const int32_t* d_track_start, const int32_t* d_members, int n_members,
                          const ps_triangulate_params* prm, ps_track_point* d_points, uint8_t* d_obs_mask, float* d_obs_error,
                          ps_triangulate_counts* counts);

#ifdef __cplusplus
}
#endif

#endif
