/* View-graph cleaning (an addition to the reference's interface): drop the relative poses that fail rotation loop
 * consistency over the triangles of the view graph, before rotation averaging, as global structure-from-motion systems
 * do (OpenMVG's rotation triplets, Theia's FilterViewGraphCyclesByRotation, the loop constraints of Zach et al.).
 *
 * ps_rotation_averaging starts from a maximum spanning tree by n_front, so a wrong relative rotation that many points
 * agree with (repeated structure, symmetric facades, an essential matrix accepted on a few points) enters the start and
 * IRLS does not recover.  For every triangle (a, b, c) of the view graph the composed rotation R(c->a) R(b->c) R(a->b)
 * should be the identity; a pair whose triangles do not close is dropped.  The output feeds ps_rotation_averaging: the kept
 * pairs' (l, r) list with d_kept.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_VIEWGRAPH_H
#define POPSIFT_B200_VIEWGRAPH_H

#include "popsift_b200_pose.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_view_graph_params {  /* 32 bytes */
    int32_t min_inliers;               /* a pair is used when n_front >= min_inliers (ps_rotation_averaging's step 1); >= 0 */
    int32_t min_consistent;            /* a tested pair is kept when n_consistent >= min_consistent ...; >= 0            */
    int32_t keep_untested;             /* 0 / 1: the fate of a used pair that lies in no triangle                          */
    int32_t pad_;                      /* ignored                                                                          */
    double  max_cycle_error;           /* degrees; a triangle is consistent when its cycle error <= this; finite, >= 0     */
    double  min_fraction;              /* ... and n_consistent >= min_fraction * n_triangles; in [0, 1]                    */
} ps_view_graph_params;

typedef struct ps_cycle_stats {        /* 12 bytes, one per pair */
    int32_t n_triangles;               /* triangles the pair lies in                                                       */
    int32_t n_consistent;              /* of those, the ones with a cycle error <= max_cycle_error                         */
    float   min_error;                 /* the smallest cycle error of those triangles, degrees; +inf when there is none    */
} ps_cycle_stats;

typedef struct ps_view_graph_report {  /* 32 bytes, HOST */
    int64_t n_triangles;               /* triangles of the graph of used pairs                                             */
    int64_t n_consistent_triangles;    /* of those, the consistent ones                                                    */
    int32_t n_used;                    /* used pairs (step 1)                                                              */
    int32_t n_kept;                    /* kept pairs (step 5)                                                              */
    int32_t n_untested;                /* used pairs that lie in no triangle                                               */
    int32_t pad_;
} ps_view_graph_report;

/* View-graph filter.  pairs (HOST, 2 per pair: l, r, each in [0, n_sets)) and d_two_view (DEVICE, one ps_two_view per
 * pair, what ps_relative_pose_batch wrote: X_r = R_p X_l + t_p), the arguments of ps_rotation_averaging.
 *   1. Used pairs: exactly ps_rotation_averaging's step 1 (n_front >= min_inliers, every entry of R_p finite, l != r).  The
 *      float R_p of a used pair is made orthonormal by gl_orthonormal (k_global.h), so that this filter and rotation
 *      averaging see the same rotation.
 *   2. Duplicates are refused: two pairs of the list that join the same two sets, in either order, give PS_ERR_ARG (a host
 *      check before any device work), so that the three pairs of a triangle are well defined.
 *   3. Triangles: an unordered triple of distinct sets {a, b, c} in which every two sets are joined by a used pair.  With
 *      the sets named so that a < b < c, and R(x->y) = R_p when pair p is stored as (x, y), R_p^T when it is stored as
 *      (y, x), the cycle error is e = |gl_log(R(c->a) (R(b->c) R(a->b)))| in degrees, all arithmetic in double in exactly
 *      that order (k_viewgraph.h: vg_cycle_error).  It does not depend on how the triangle was found, nor on which way its
 *      pairs are stored.
 *   4. Per-pair statistics (ps_cycle_stats): n_triangles, n_consistent (the triangles with e <= max_cycle_error) and
 *      min_error (the smallest e, rounded to float).  Unused pairs: 0, 0, +inf.
 *   5. Decision, in one pass over the full graph of used pairs (dropping a pair does not re-test the others):
 *        a used pair with n_triangles > 0 is kept when n_consistent >= min_consistent and
 *        (double)n_consistent >= min_fraction * (double)n_triangles;
 *        a used pair with n_triangles == 0 is kept when keep_untested is 1;
 *        an unused pair is never kept.
 *   6. Outputs.  keep (HOST, a byte per pair, 0 or 1); stats (HOST, optional, a ps_cycle_stats per pair); d_kept (DEVICE,
 *      optional): the kept pairs' ps_two_view records, byte for byte, compacted in pair order (n_kept records).  The kept
 *      pairs' (l, r) list with d_kept is the input of ps_rotation_averaging.  *report: the totals.
 *   7. Determinism: only integer atomics (the counts are sums, min_error an atomicMin on the bit pattern of a non-negative
 *      float); the results do not depend on the order of the updates, and two identical calls give identical bytes.
 * Errors: PS_ERR_ARG, with no output written, for n_sets or n_pairs < 0; prm, keep or report NULL; pairs NULL with
 * n_pairs > 0, or an index outside [0, n_sets); a duplicate pair; d_two_view not device memory on `device` with
 * n_pairs > 0; a non-NULL d_kept that is not device memory on `device`; a parameter outside its range above.  n_sets = 0
 * and n_pairs = 0 are valid.  Synchronous; one read-back of keep, stats and the totals.
 * Workspace from the library's memory pool: 113 bytes per pair (its ends, orthonormal rotation, statistics, flag and
 * position, the two sort keys and the two sort buffers), 4 bytes per adjacency entry (one per pair: a used pair is one
 * oriented entry), 8 bytes per set (its degree and its out-list offset), plus the scan and sort scratch (about 1 KB per
 * 4 096 pairs). */
int ps_view_graph_filter(int device, int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view,
                         const ps_view_graph_params* prm, uint8_t* keep, ps_cycle_stats* stats, ps_two_view* d_kept,
                         ps_view_graph_report* report);

#ifdef __cplusplus
}
#endif

#endif
