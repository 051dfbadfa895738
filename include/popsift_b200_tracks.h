/* Feature tracks (an addition to the reference's interface): the connected components of verified matches across all
 * pairs of a set of images, with conflicting components dropped.
 *
 * A structure-from-motion back end consumes tracks: each physical 3-D point seen as one keypoint in each of several
 * images.  OpenMVG / AliceVision's TracksBuilder forms them as the union-find of all pairwise inlier matches, drops every
 * track that holds two features of one image (a fork) and every track shorter than a minimum length.  These entry points
 * do that on the device, so that the chain extract -> ps_retrieve_pairs -> ps_match_batch -> ps_match_correspondences ->
 * ps_verify_batch (-> ps_match_guided_batch) -> tracks never leaves it; only the tracks come back.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_TRACKS_H
#define POPSIFT_B200_TRACKS_H

#include "popsift_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Nodes.  A node is a feature (a Feature record of ps_download / ps_download_dev), not a descriptor: the up to four
 * orientations of one keypoint are one 2-D point.  Set i has n_feat[i] features (a host array); the global id of feature
 * f of set i is off[i] + f with off[i] = sum_{j<i} n_feat[j], and N = sum n_feat[i] must be < 2^31.
 *
 * Components.  Connected components are taken over all edges; self-loops (u == v) are ignored, and duplicate edges and
 * both directions of an edge are allowed.  A component is a set of >= 2 features joined by edges.  It is conflicting when
 * two of its features belong to one set, and is then dropped whole; a non-conflicting component with fewer than
 * min_length features is short, and is dropped too (min_length >= 2).  The survivors are the tracks.
 *
 * Outputs (DEVICE, on `device`; capacities from N alone):
 *   d_track_of[N]                          every feature's track index, or -1;
 *   d_track_start[n_tracks + 1]            capacity N / min_length + 1: track t's members are
 *   d_members[n_members]                   capacity N: d_members[d_track_start[t] .. d_track_start[t + 1] - 1], global ids;
 *   *counts (HOST)                         the five counts below.
 * Order (the determinism contract): tracks are sorted by their smallest member id; members within a track ascend by
 * global id, that is by set, since a track has at most one feature per set.  The output depends only on the set of
 * distinct non-loop edges, not on their order, duplicates or direction; two identical calls give identical bytes.
 *
 * Errors.  An endpoint outside [0, N) (for ps_tracks_from_matches: a row, match or reverse-map index outside its set) is
 * found on the device: a flag is read back before anything is written to the outputs, and the call returns PS_ERR_ARG with
 * the outputs untouched.  Also PS_ERR_ARG: n_sets < 0, a negative count, N >= 2^31, min_length < 2, a null pointer where a
 * count is > 0, counts == NULL, or an array that is not device memory on `device` (d_track_start always; d_track_of and
 * d_members when N > 0).
 *
 * Workspace comes from the matcher's memory pool: 24 bytes per feature, plus 1 / 16 byte per feature for the radix
 * histograms, 4 bytes per set and, for ps_tracks_from_matches, 64 bytes per pair with correspondences.  Edges take no
 * workspace: both entry points read them where they are. */
typedef struct ps_track_counts {      /* 20 bytes */
    int32_t n_tracks;        /* tracks kept                                                        */
    int32_t n_members;       /* features in them: d_track_start[n_tracks]                          */
    int32_t n_components;    /* components of >= 2 features                                        */
    int32_t n_conflicting;   /* components dropped for two features of one set                     */
    int32_t n_short;         /* non-conflicting components dropped for fewer than min_length       */
} ps_track_counts;

/* Tracks of an explicit edge list: d_edges (DEVICE) holds n_edges pairs (u, v) of global ids, 2 x int32 each.
 * n_edges = 0 is valid and gives no tracks. */
int ps_tracks_from_edges(int device, int n_sets, const int32_t* n_feat, int n_edges, const int32_t* d_edges, int min_length,
                         int32_t* d_track_of, int32_t* d_track_start, int32_t* d_members, ps_track_counts* counts);

/* Tracks of the verification chain's own device arrays, without an edge list.  pairs, n_desc and d_match are what
 * ps_match_batch / ps_match_u8_batch / ps_match_guided_batch took and gave; d_src and n_corr what ps_match_correspondences
 * gave for them; d_rev[i] the descriptor -> feature reverse map of set i (ps_download_dev); d_inlier_mask what
 * ps_verify_batch gave, or NULL for every correspondence (the rows of guided matching already passed the model).
 * pairs, n_desc, n_feat, n_corr and d_rev are host arrays.  Pair p = (l, r)'s rows start at start_p = sum_{q<p}
 * n_desc[pairs[2q]]; for k = start_p .. start_p + n_corr[p] - 1 with d_inlier_mask[k] != 0 (or no mask):
 *     i = d_src[k],  b = d_match[3 (start_p + i)],  edge = (off[l] + d_rev[l][i], off[r] + d_rev[r][b])
 * A self pair (i, i) is valid; its edges join features of one set, so they make their component conflicting unless they
 * are self-loops.  Also PS_ERR_ARG: what ps_match_correspondences refuses, and n_corr[p] outside [0, n_desc[pairs[2p]]]. */
int ps_tracks_from_matches(int device, int n_sets, const int32_t* n_feat, const int32_t* const* d_rev, const int32_t* n_desc,
                           int n_pairs, const int32_t* pairs, const int32_t* d_match, const int32_t* d_src, const int32_t* n_corr,
                           const uint8_t* d_inlier_mask, int min_length, int32_t* d_track_of, int32_t* d_track_start,
                           int32_t* d_members, ps_track_counts* counts);

#ifdef __cplusplus
}
#endif

#endif
