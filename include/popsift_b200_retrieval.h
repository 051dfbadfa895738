/* Image retrieval (an addition to the reference's interface): which pairs of a large image set are worth matching.
 *
 * Matching every ordered pair of N images grows as N^2, and almost all of those pairs share no content.  SfM front ends
 * give every image a global descriptor and match each image only with its m most similar ones (COLMAP's vocabulary-tree
 * matching, the NetVLAD / VLAD shortlists of hloc).  These entry points do that on the device:
 *   ps_vlad_train     a k-means codebook of SIFT descriptors (the visual words);
 *   ps_vlad_encode    one VLAD vector per image (and each descriptor's visual word);
 *   ps_retrieve_pairs all-vs-all inner products with each image's m best neighbours, the pair list for ps_match_batch.
 * The chain extract -> ps_vlad_encode -> ps_retrieve_pairs -> ps_match_batch -> ps_verify_batch never leaves the device.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_RETRIEVAL_H
#define POPSIFT_B200_RETRIEVAL_H

#include "popsift_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Sets.  d_sets[i] (DEVICE, on `device`) holds n_desc[i] descriptors; d_sets and n_desc are host arrays, as in
 * ps_match_batch.  The pool is the concatenation of the sets in set order, N = sum n_desc[i] descriptors.
 *
 * Assignment.  Descriptor x goes to the centroid of smallest squared L2 distance: the `best` column of
 * ps_match_batch(x's set, centroids, flags), ties to the lower index.  flags: PS_MATCH_AUTO / EXACT / TENSOR as there
 * (PS_MATCH_EXACT is the CUDA-core scan; the tensor path carries ps_match_batch's near-tie caveat). */

/* k-means codebook: d_centroids (DEVICE, k x 128 floats) is written.
 * Initialisation: key = verify_mix(seed) (splitmix64's finaliser, the sample hash of ps_verify_batch); draw c = 0, 1, 2, ...
 * is pool index ((verify_mix(key + c) >> 32) * N) >> 32, repeats skipped, until k indices are distinct; centroid i is the
 * pool row of the i-th distinct index.  iters = 0 returns exactly these rows.
 * Iteration (exactly `iters`, no convergence test): assign every pool descriptor, then centroid c = the mean of its
 * members, summed in double: every chunk of up to 2 048 consecutive descriptors of one set is summed in descriptor order
 * from zero, and the chunks' sums are added in pool order in one chain from zero, whatever the grouping of the sets (see
 * ps_vlad_encode); the mean is rounded once to float after the division.  A centroid without members keeps its value.
 * PS_ERR_ARG for what ps_match_batch refuses, k outside [1, 1024], iters outside [0, 1000], N < k, N >= 2^31, or
 * d_centroids that is not device memory on `device`. */
int ps_vlad_train(int device, int n_sets, const ps_descriptor* const* d_sets, const int32_t* n_desc, int k, int iters,
                  uint64_t seed, float* d_centroids, int flags);

/* VLAD vectors: row i of d_vlad (DEVICE, n_sets x k*128 floats) is set i's encoding under the codebook d_centroids
 * (DEVICE, k x 128 floats).
 *   V[c] = sum over the set's descriptors x assigned to c of (x - mu_c), in double, in descriptor order (chunks, as above);
 *   each 128-block divided by its L2 norm (an all-zero block stays zero), then sign(v) sqrt(|v|), then the whole vector
 *   divided by its L2 norm; all in double, written as float.  An empty set gives a zero row.
 * d_assign (DEVICE, optional, NULL allowed): one int32 per pool descriptor, its centroid (visual word).
 * Workspace comes from the matcher's pool; both VLAD entry points process the sets in groups under POPSIFT_B200_MATCH_WS
 * (default 1 GB), and their results do not depend on the grouping.
 * PS_ERR_ARG for what ps_match_batch refuses, k outside [1, 1024], and d_centroids / d_vlad / a non-NULL d_assign that
 * is not device memory on `device`.  n_sets = 0 is valid. */
int ps_vlad_encode(int device, int n_sets, const ps_descriptor* const* d_sets, const int32_t* n_desc, int k,
                   const float* d_centroids, float* d_vlad, int32_t* d_assign, int flags);

/* Nearest neighbours of n vectors under the inner product.  d_vec (DEVICE, 16-byte aligned): n rows of `dim` floats,
 * dim > 0 and a multiple of 4.
 * Score: score(i, j) is  acc = 0; for d = 0 .. dim-1: acc = fmaf(v_i[d], v_j[d], acc)  in float32, so
 * score(i, j) == score(j, i) bit for bit.
 * Output: d_nbr (int32) and d_score (float), DEVICE, n x m each: row i holds the m largest scores over j != i in
 * descending order, equal scores to the lower j (+0 and -0 are equal), NaN below every number.  Slots beyond n - 1 hold
 * j = -1 and score -inf.  Results depend only on the input.
 * PS_ERR_ARG for n < 0, dim <= 0 or not a multiple of 4, m outside [1, 128], and (n > 0) d_vec not 16-byte aligned or any
 * array that is not device memory on `device`.  n = 0 is valid. */
int ps_retrieve_pairs(int device, int n, const float* d_vec, int dim, int m, int32_t* d_nbr, float* d_score);

#ifdef __cplusplus
}
#endif

#endif
