/*
 * popsift_b200 -- C ABI of the H100-native (sm_90a) SIFT extractor.
 *
 * This is the drop-in boundary for the hot path of alicevision/popsift:
 *     image -> Gaussian pyramid -> DoG extrema -> orientation -> descriptors.
 * The reference has no C ABI; its boundary for this path is the C++ class
 * popsift::Pyramid (reference src/popsift/sift_pyramid.h:88-114:
 * step1 / step2 / get_descriptors / clone_device_descriptors) driven by
 * PopSift::extractDownloadLoop (src/popsift/popsift.cpp:306-344).  Each entry
 * point below names the reference interface it replaces.
 *
 * Conventions: plain pointers and sizes, no C++ types, nothing throws across
 * the ABI.  Functions return 0 (PS_OK) or a negative ps_status; the message
 * is available from ps_last_error().  A context belongs to one CUDA device;
 * its slots are independent in-flight images (one CUDA stream each).
 * There is NO CPU fallback: without a usable CUDA device ps_create fails.
 */
#ifndef POPSIFT_B200_H
#define POPSIFT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PS_ABI_VERSION   3
#define PS_MAX_OCTAVES   20   /* reference sift_conf.h:12  MAX_OCTAVES   */
#define PS_GAUSS_ALIGN   32   /* reference sift_constants.h:37            */
#define PS_GAUSS_LEVELS  12   /* reference sift_constants.h:38            */
#define PS_MAX_ORI       4    /* reference sift_constants.h:54            */
#define PS_MAX_FILTER_GRID 32 /* grid filter: at most 32 x 32 cells        */

typedef enum ps_status {
    PS_OK             =  0,
    PS_ERR_ARG        = -1,  /* bad argument / unsupported configuration        */
    PS_ERR_CUDA       = -2,  /* a CUDA call failed (message in ps_last_error)   */
    PS_ERR_TOO_LARGE  = -3,  /* image exceeds the size the context was made for */
    PS_ERR_STATE      = -4,  /* call order (e.g. download before submit)        */
    PS_ERR_OVERFLOW   = -5   /* more extrema/descriptors than the slot capacity */
} ps_status;

/* enum values follow reference sift_conf.h:33-107 */
enum { PS_MODE_POPSIFT = 0, PS_MODE_OPENCV = 1, PS_MODE_VLFEAT = 2 };
enum { PS_GAUSS_VLFEAT_COMPUTE = 0, PS_GAUSS_VLFEAT_RELATIVE = 1, PS_GAUSS_VLFEAT_RELATIVE_ALL = 2,
       PS_GAUSS_OPENCV_COMPUTE = 3, PS_GAUSS_FIXED9 = 4, PS_GAUSS_FIXED15 = 5 };
enum { PS_DESC_LOOP = 0, PS_DESC_ILOOP = 1, PS_DESC_GRID = 2, PS_DESC_IGRID = 3, PS_DESC_NOTILE = 4 };
enum { PS_NORM_ROOTSIFT = 0, PS_NORM_CLASSIC = 1 };
enum { PS_SCALE_DIRECT = 0, PS_SCALE_DEFAULT = 1 };                                  /* sift_conf.h:75-80   */
enum { PS_FILTER_RANDOM = 0, PS_FILTER_LARGEST_FIRST = 1, PS_FILTER_SMALLEST_FIRST = 2 }; /* sift_conf.h:118-125 */

/* The fields of popsift::Config (reference sift_conf.h:29-409) that the kernels consume. */
typedef struct ps_config {
    int32_t octaves;           /* -1 = auto (popsift.cpp:118-122)                         */
    int32_t levels;            /* 3; clamped to >= 2 (popsift.cpp:86)                      */
    float   sigma;             /* 1.6                                                      */
    float   edge_limit;        /* 10                                                       */
    float   threshold;         /* 0.04 (peak threshold = thr*0.5*255/levels)               */
    float   upscale;           /* 1.0 = -downsampling                                      */
    float   initial_blur;      /* 0.5                                                      */
    int32_t has_initial_blur;  /* 1                                                        */
    int32_t sift_mode;         /* PS_MODE_*                                                */
    int32_t gauss_mode;        /* PS_GAUSS_*  (all six; FIXED9 / FIXED15 need levels == 3 like the reference) */
    int32_t desc_mode;         /* PS_DESC_*   (loop is the fast path; iloop / grid / igrid / notile follow the reference's schemes) */
    int32_t norm_mode;         /* PS_NORM_*                                                */
    int32_t norm_multi;        /* descriptor scaled by 2^norm_multi                        */
    int32_t max_extrema;       /* 100000 per octave                                        */
    /* ABI 2 */
    int32_t scaling_mode;      /* PS_SCALE_*  (DIRECT: level 0 of every octave straight from the input image)         */
    int32_t filter_max_extrema;/* <= 0: grid filter off (reference sift_conf.cu:30, s_orientation.cu:380-383)        */
    int32_t filter_grid_size;  /* 2: cells per image side (s_filtergrid.cu:125)                                      */
    int32_t filter_sort;       /* PS_FILTER_*                                                                        */
} ps_config;

/* Same bytes as popsift::Descriptor (reference sift_extremum.h:69-72). */
typedef struct ps_descriptor { float features[128]; } ps_descriptor;

/* Same bytes as popsift::Feature (reference features.h:23-37), 72 bytes. */
typedef struct ps_feature {
    int32_t        debug_octave;
    float          xpos, ypos, sigma;
    int32_t        num_ori;
    float          orientation[PS_MAX_ORI];
    int32_t        pad_;
    ps_descriptor* desc[PS_MAX_ORI];   /* host pointers into the array given to ps_download */
} ps_feature;

/* Internal extremum record, exposed for tests (octave-local coordinates). */
typedef struct ps_extremum {
    float   xpos, ypos;
    int32_t lpos;
    float   sigma;
    int32_t octave, num_ori, idx_ori;
    float   orientation[PS_MAX_ORI];
} ps_extremum;

typedef struct ps_gauss_tables {
    float   inc_filter[PS_GAUSS_LEVELS * PS_GAUSS_ALIGN];  /* gauss_filter.cu:173-188 */
    float   inc_sigma[PS_GAUSS_LEVELS];
    int32_t inc_span[PS_GAUSS_LEVELS];
    float   dd_filter0[PS_GAUSS_ALIGN];                    /* gauss_filter.cu:227-238, octave 0 */
    float   dd_sigma0;
    int32_t dd_span0;
    float   peak_threshold;                                /* sift_conf.cu:276-279 */
    float   sigma_k;                                       /* sift_constants.cu:27 */
    /* ABI 3: the direct-downscaling rows of every octave (gauss_filter.cu:216-238), used by Config::ScaleDirect:
     * level 0 of octave o is filtered horizontally with row o straight from the input image.  Row 0 == dd_filter0. */
    float   dd_filter[PS_MAX_OCTAVES * PS_GAUSS_ALIGN];
    float   dd_sigma[PS_MAX_OCTAVES];
    int32_t dd_span[PS_MAX_OCTAVES];
    /* the absolute rows of octave 0 (gauss_filter.cu:190-199), used by --gauss-mode vlfeat-direct (VLFeat_Relative_All):
     * every level of octave 0 is filtered straight from the input image with row `level`, horizontally and vertically */
    float   abs_filter[PS_GAUSS_LEVELS * PS_GAUSS_ALIGN];
    float   abs_sigma[PS_GAUSS_LEVELS];
    int32_t abs_span[PS_GAUSS_LEVELS];
    /* the incremental rows transformed for hardware interpolation (gauss_filter.cu:372-405), used by --gauss-mode relative
     * (= vlfeat-hw-interpolated, VLFeat_Relative): [0] centre weight, odd x: fraction u, even x: pair weight v */
    float   inc_ifilter[PS_GAUSS_LEVELS * PS_GAUSS_ALIGN];
    int32_t inc_ispan[PS_GAUSS_LEVELS];
    /* the absolute rows of octaves >= 1 (gauss_filter.cu:200-214): level l straight from level 0 of the same octave; used by
     * --gauss-mode fixed9 / fixed15 */
    float   absn_filter[PS_GAUSS_LEVELS * PS_GAUSS_ALIGN];
    float   absn_sigma[PS_GAUSS_LEVELS];
    int32_t absn_span[PS_GAUSS_LEVELS];
} ps_gauss_tables;

enum { PS_STAGE_H2D = 0, PS_STAGE_PYRAMID = 1, PS_STAGE_EXTREMA = 2, PS_STAGE_ORIENT = 3,
       PS_STAGE_DESC = 4, PS_STAGE_TOTAL = 5, PS_NUM_STAGES = 6 };
enum { PS_PLANE_GAUSS = 0, PS_PLANE_DOG = 1 };

typedef struct ps_ctx ps_ctx;

/* ---- host-only helpers: usable without a GPU -------------------------------------------- */

int  ps_abi_version(void);
/* popsift::Config::Config() defaults (reference sift_conf.cu:18-41) */
void ps_config_default(ps_config* cfg);
/* replaces init_filter + init_constants (reference gauss_filter.cu:127-257, sift_constants.cu:22-53) */
int  ps_gauss_tables_compute(const ps_config* cfg, ps_gauss_tables* out);
/* replaces the printout of Config::setPrintGaussTables() / --print-gauss-tables (gauss_filter.cu:24-121,146-161,247-256): the
 * same text, from this library's tables.  Returns the text length; writes at most cap - 1 characters + 0 into buf (may be NULL) */
int  ps_format_gauss_tables(const ps_config* cfg, char* buf, size_t cap);
/* replaces PopSift::private_apply_scale_factor + Pyramid ctor geometry
 * (reference popsift.cpp:109-126, sift_pyramid.cu:129-134); returns #octaves or <0 */
int  ps_geometry(const ps_config* cfg, int w, int h, int32_t* W, int32_t* H);

/* ---- device path ------------------------------------------------------------------------ */

/* replaces PopSift ctor + Pyramid ctor (reference popsift.cpp:25-48,128-144; sift_pyramid.cu:108-159):
 * allocates n_slots independent pipelines for images up to max_w x max_h on `device`. */
ps_ctx* ps_create(int device, const ps_config* cfg, int max_w, int max_h, int n_slots);
/* replaces Pyramid dtor / PopSift::uninit (reference sift_pyramid.cu:211-225) */
void    ps_destroy(ps_ctx* ctx);
/* last error text; ctx may be NULL for ps_create failures */
const char* ps_last_error(const ps_ctx* ctx);

/* replaces SiftJob::setImg/Image::load + Pyramid::step1 + step2
 * (reference popsift.cpp:293-344,432-437; s_image.cu:69-77; sift_pyramid.cu:227-240):
 * copies the host image to the device and enqueues every kernel of the hot path on the slot's
 * stream.  Returns without waiting for the GPU.
 * Lifetime of `host_img`: a PAGEABLE buffer is copied before the call returns and may be reused or
 * freed at once.  A PAGE-LOCKED buffer (ps_host_alloc, cudaHostAlloc, cudaHostRegister) is read by an
 * asynchronous DMA: it must stay valid and unmodified until ps_wait_input(), ps_counts() or ps_sync()
 * has returned for this slot. */
int ps_submit_u8 (ps_ctx* ctx, int slot, const uint8_t* host_img, int w, int h);
/* float images, value range [0,1) (reference popsift.h:62-69, s_image.cu:262-291) */
int ps_submit_f32(ps_ctx* ctx, int slot, const float* host_img, int w, int h);
/* same, input already resident in device memory (pitch in bytes); no host copy */
int ps_submit_dev_u8(ps_ctx* ctx, int slot, const uint8_t* dev_img, size_t pitch, int w, int h);

/* replaces Pyramid::readDescCountersFromDevice (reference sift_pyramid.cu:371-379):
 * waits for the slot, returns the number of features and descriptors. */
int ps_counts(ps_ctx* ctx, int slot, int32_t* n_feat, int32_t* n_desc);
/* replaces Pyramid::get_descriptors + prep_features (reference sift_pyramid.cu:250-322):
 * copies n_feat Feature records and n_desc descriptors to the caller's arrays; Feature::desc[]
 * are host pointers into `desc`. */
int ps_download(ps_ctx* ctx, int slot, ps_feature* feat, ps_descriptor* desc);
/* replaces Pyramid::clone_device_descriptors (reference sift_pyramid.cu:324-362), the result path of
 * Config::MatchingMode: copies the slot's n_feat Feature records, n_desc descriptors and the
 * descriptor -> feature reverse map into caller-owned DEVICE arrays (sizes from ps_counts);
 * Feature::desc[] are device pointers into `d_desc`.  Nothing is copied to the host. */
int ps_download_dev(ps_ctx* ctx, int slot, ps_feature* d_feat, ps_descriptor* d_desc, int32_t* d_rev);
/* device memory for ps_download_dev results (thin wrappers of cudaMalloc / cudaFree on the current
 * device) and a blocking device -> host copy for callers without a CUDA toolchain */
void* ps_dev_alloc(size_t bytes);
void  ps_dev_free(void* p);
int   ps_dev_to_host(void* dst_host, const void* src_dev, size_t bytes);
int   ps_host_to_dev(void* dst_dev, const void* src_host, size_t bytes);
/* ordinal of the CUDA device a device pointer belongs to, or -1 */
int   ps_pointer_device(const void* dev_ptr);
/* replaces FeaturesDev::match -> compute_distance (reference features.cu:165-227,282-304): brute-force 2-nearest-
 * neighbour search of every LEFT descriptor among the RIGHT descriptors by squared L2 distance.  d_left / d_right are
 * DEVICE arrays (e.g. the descriptor arrays filled by ps_download_dev); d_out receives n_left x {best index, second
 * index, accept} with accept = (best / second < 0.8f), also in DEVICE memory.  The call returns when the result is
 * complete.  flags: PS_MATCH_AUTO, or force one implementation (PS_MATCH_EXACT: CUDA cores in the reference's
 * evaluation order; PS_MATCH_TENSOR: wgmma tf32x3 candidate pass + exact re-rank). */
enum { PS_MATCH_AUTO = 0, PS_MATCH_EXACT = 1, PS_MATCH_TENSOR = 2 };
int ps_match(int device, const ps_descriptor* d_left, int n_left, const ps_descriptor* d_right, int n_right,
             int32_t* d_out, int flags);
/* 2-NN matching of many pairs of descriptor sets in one call (an addition to the reference's interface).  d_sets[i]
 * (DEVICE, on `device`, n_desc[i] descriptors) for i < n_sets; pairs = n_pairs x {left set, right set} (i == j allowed).
 * d_sets, n_desc and pairs are host arrays.  d_out (DEVICE) receives, for pair p, n_desc[pairs[2p]] rows {best, second,
 * accept} starting at row sum_{q<p} n_desc[pairs[2q]]: row by row what ps_match(device, d_sets[l], n_desc[l], d_sets[r],
 * n_desc[r], ..., flags) gives.  Empty left sets contribute no rows; an empty right set gives rows (0, 0, 0).
 * PS_MATCH_EXACT runs the CUDA-core kernel pair by pair; PS_MATCH_AUTO / PS_MATCH_TENSOR split every set once per group
 * of pairs and run all pairs' tensor-core work in one persistent launch, then one re-rank launch.  Returns when the
 * result is complete; PS_ERR_ARG for negative counts, a set index out of range, a null pointer with a count > 0, or a
 * set that is not device memory on `device`. */
int ps_match_batch(int device, int n_sets, const ps_descriptor* const* d_sets, const int32_t* n_desc,
                   int n_pairs, const int32_t* pairs, int32_t* d_out, int flags);
/* Device-side quantisation of float descriptors to 8 bits (an addition to the reference's interface):
 * d_out[128 i + k] = roundf(min(max(d_in[i].features[k], 0), 255)), NaN -> 0.  For components in [0, 255] this is the
 * value the reference prints under --write-as-uchar (features.cu:317-320); larger values saturate.  Scaling is the
 * caller's, e.g. ps_config::norm_multi = 9 as the reference's help text suggests.  d_in (n descriptors) and d_out
 * (n x 128 bytes) are DEVICE memory on `device`.  Returns when the result is complete; PS_ERR_ARG for n < 0, a null
 * pointer with n > 0, or a pointer that is not device memory on `device`. */
int ps_descriptors_to_u8(int device, const ps_descriptor* d_in, int n, uint8_t* d_out);
/* ps_match_batch for 8-bit descriptors: d_sets[i] = n_desc[i] rows of 128 uint8_t (DEVICE, on `device`, 16-byte
 * aligned).  Same pair list, output layout and argument checks as ps_match_batch, and a set pointer that is not 16-byte
 * aligned is refused with PS_ERR_ARG.  Distances are exact integers: pair p's rows are bit for bit what
 * ps_match_batch(..., PS_MATCH_EXACT) gives on float32 copies of the same sets -- best = the smallest (distance, index),
 * second = the next, accept = float(d1) / float(d2) < 0.8f (equal distances give 0); an empty right set gives (0, 0, 0),
 * a single right descriptor (0, 0, 1).  PS_MATCH_AUTO / PS_MATCH_TENSOR run the integer tensor-core path (wgmma u8 x u8
 * -> s32), PS_MATCH_EXACT a CUDA-core kernel pair by pair. */
int ps_match_u8_batch(int device, int n_sets, const uint8_t* const* d_sets, const int32_t* n_desc,
                      int n_pairs, const int32_t* pairs, int32_t* d_out, int flags);

/* ---- geometric verification of matched pairs (an addition to the reference's interface): correspondences from the rows
 * of ps_match_batch / ps_match_u8_batch, then one RANSAC homography or fundamental matrix per pair, all on the device. */

/* Point correspondences of matched pairs.  Per set i < n_sets (host arrays): d_feat[i] / d_rev[i] are the Feature records
 * and the descriptor -> feature reverse map of ps_download_dev (DEVICE, on `device`), n_desc[i] the descriptor count.  pairs
 * and d_match are exactly what ps_match_batch / ps_match_u8_batch took and gave (both write the same row layout).  For
 * pair p = (l, r), left descriptor row i with accept == 1 and best = b gives the correspondence
 *     d_corr[4 k ..] = (feat_l[rev_l[i]].xpos, .ypos, feat_r[rev_r[b]].xpos, .ypos),   d_src[k] = i
 * except that row i is dropped when an accepted row i' with i - 3 <= i' < i has rev_l[i'] == rev_l[i] and
 * rev_r[best_i'] == rev_r[b] (the up to four orientations of one Feature matching the same point).  Pair p's
 * correspondences keep row order and start at row sum_{q<p} n_desc[pairs[2q]] of d_corr / d_src (DEVICE, float4 / int32
 * per row, as many rows as d_match has); their number goes to the HOST array n_corr[p].  A pair with an empty right set
 * gives none.  Returns when the result is complete; PS_ERR_ARG for negative counts, a set index out of range, a null
 * pointer where a count is > 0, or a pointer that is not device memory on `device`.  Empty sets and self pairs are valid. */
int ps_match_correspondences(int device, int n_sets, const ps_feature* const* d_feat, const int32_t* const* d_rev,
                             const int32_t* n_desc, int n_pairs, const int32_t* pairs, const int32_t* d_match,
                             float* d_corr, int32_t* d_src, int32_t* n_corr);

enum { PS_GEOM_HOMOGRAPHY = 0, PS_GEOM_FUNDAMENTAL = 1 };
typedef struct ps_verify_params {      /* 24 bytes */
    int32_t  model;       /* PS_GEOM_*                                                         */
    int32_t  n_samples;   /* minimal samples per pair, 1 .. 65536 (fixed; no early exit)        */
    float    threshold;   /* pixels, input-image units; finite and > 0                          */
    int32_t  refine;      /* 1: one least-squares refit on the winner's inliers; 0: none        */
    uint64_t seed;
} ps_verify_params;
/* test tap: when given, every hypothesis's inlier count (-1: invalid) and its model in pixels (scaled like the output
 * model, zero when invalid); pair p's block starts at hypothesis p * k * n_samples (k below) */
typedef struct ps_verify_taps { int32_t* d_counts; float* d_models; } ps_verify_taps;
/* Batched RANSAC.  Pair p's correspondences are rows corr_start[p] .. corr_start[p] + n_corr[p] - 1 of d_corr (DEVICE,
 * 4 floats per row: x_l, y_l, x_r, y_r in pixels; 16-byte aligned); corr_start, n_corr and prm are host memory.
 *   Normalisation: c_l, c_r = the means of the left / right points, d = (sum |x_l - c_l| + sum |x_r - c_r|) / 2n,
 *     s = sqrt(2) / d (1 when d == 0), all in double; a point becomes s (x - c) in float32.  One scale for both images, so
 *     the transfer error and the Sampson distance scale by exactly s and the test below runs against (s t)^2.
 *   Error and inlier test, in normalised float32 coordinates, without division:
 *     homography (one-sided transfer error in the right image, as cv::findHomography): (u, v, w) = H x_l,
 *       inlier when (u - x_r w)^2 + (v - y_r w)^2 < (s t)^2 w^2;
 *     fundamental (Sampson distance of x_r^T F x_l = 0): a = F x_l, b = F^T x_r, e = x_r . a,
 *       inlier when e^2 < (s t)^2 (a0^2 + a1^2 + b0^2 + b1^2).
 *   Samples: sample s of pair p draws m = 4 (H) or 7 (F) distinct indices into the pair's n correspondences with
 *       mix(z)  = z += 0x9E3779B97F4A7C15; z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9; z = (z ^ z >> 27) * 0x94D049BB133111EB;
 *                 z ^ z >> 31                                                  (splitmix64, uint64 arithmetic)
 *       key     = mix(seed ^ mix((uint64)p << 32 | s))
 *       draw c  = (uint32)(((mix(key + c) >> 32) * n) >> 32),   c = 0, 1, .., 63
 *     taking draws in order and skipping repeated indices; a sample without m distinct indices after 64 draws is invalid.
 *   Hypotheses: h = k s + root with k = 1 (H) or 3 (F).  H: the 4-point DLT; the sample is rejected when three of its
 *     points are collinear in either image (|(b - a) x (c - a)| < 1e-7 in normalised coordinates).  F: the 7-point method,
 *     F = lambda F1 + (1 - lambda) F2 over the sample's null space, up to three real roots of det F = 0 in ascending
 *     lambda; a missing root or a failed solve (null space not two-dimensional) gives an invalid hypothesis.
 *   Selection: the hypothesis with the most inliers wins, ties to the smallest h; invalid hypotheses never win.
 *   Refit (refine = 1, and at least 4 (H) / 8 (F) inliers): the normalised DLT (H) or the 8-point method with rank-2
 *     enforcement (F) on the winner's inliers, the smallest eigenvector of the 9 x 9 normal matrix (double, fixed order,
 *     Jacobi); kept when its inlier count is >= the winner's.  Not iterated.
 *   Output: d_models[9 p ..] (DEVICE, row-major) maps left to right in pixels.  H is scaled to H22 = 1, or to Frobenius
 *     norm 1 when |H22| < 1e-8 of that norm; F has Frobenius norm 1 and its largest-magnitude entry positive.
 *     d_inlier_mask (DEVICE, one byte per d_corr row) is the inlier test above under the output model; d_n_inliers[p]
 *     (DEVICE) is its sum.  n < 4 (H) / 7 (F), or no valid hypothesis: zero model, count 0, mask 0 -- not an error.
 *   Determinism: results depend only on (seed, p, the pair's correspondences, prm); two identical calls give identical
 *     bytes.
 * Returns when the result is complete.  PS_ERR_ARG for an unknown model, n_samples outside [1, 65536], a threshold that is
 * not finite and > 0, refine not 0 / 1, negative counts or starts, a null pointer where a count is > 0, or a pointer that
 * is not device memory on `device`.  n_pairs = 0 is valid. */
int ps_verify_batch(int device, int n_pairs, const float* d_corr, const int32_t* corr_start, const int32_t* n_corr,
                    const ps_verify_params* prm, float* d_models, int32_t* d_n_inliers, uint8_t* d_inlier_mask,
                    const ps_verify_taps* taps);
/* ---- describe: orientations and descriptors at caller-supplied keypoints (an addition to the reference's interface;
 * VLFeat's vl_sift 'Frames' / 'Orientations', OpenCV's Feature2D::compute).  Used for tracking, upright SIFT, dense SIFT,
 * keypoints from another detector and re-describing stored keypoints under another desc_mode / norm_mode. */

/* A keypoint to describe, in input-image units exactly like ps_feature (24 bytes). */
typedef struct ps_keypoint {
    float   xpos, ypos, sigma;
    float   orientation;   /* radians; used unless PS_DESCRIBE_ORIENT */
    int32_t octave;        /* -1: derived from sigma (rule below); else the octave, as ps_feature::debug_octave */
    int32_t level;         /* -1: derived from sigma; else the Gaussian level (ps_extremum::lpos), 0 .. L+2 */
} ps_keypoint;
enum { PS_DESCRIBE_GIVEN = 0, PS_DESCRIBE_ORIENT = 1 };
/* Builds the slot's pyramid of the image (same rules as ps_submit_u8 / ps_submit_f32: lifetime, page-locked staging, size
 * checks), skips the extrema stage and the grid filter, and describes the n keypoints of the host array kps (copied
 * before the call returns).  Results are read with ps_counts / ps_download / ps_download_dev as after a submission:
 *   - one Feature per keypoint, in input order: n_feat == n, Feature i is keypoint i, with the keypoint's own xpos, ypos
 *     and sigma bits and debug_octave = the octave used (-1 for a rejected keypoint); the descriptors of Feature i follow
 *     those of Feature i - 1, and ps_download_dev's reverse map points into input order;
 *   - PS_DESCRIBE_GIVEN: num_ori = 1, orientation[0] = the given angle, one descriptor at it;
 *   - PS_DESCRIBE_ORIENT: the orientation stage runs at the keypoint (the given angle is ignored): num_ori 1 .. 4 and the
 *     angles as for a detected extremum;
 *   - a rejected keypoint keeps its place with num_ori = 0, zero angles and no descriptor (not an error).  Rejected are:
 *     a non-finite x, y or sigma (under GIVEN also angle); sigma <= 0; an explicit octave outside [0, n_octaves) or an
 *     explicit level outside [0, L+2] (any negative value other than -1 is explicit); a position outside
 *     [0, W_o - 1] x [0, H_o - 1] of its octave, where local = image * 2^(up_fac - octave) (exact);
 *   - a derived octave and level, in float32 with up_fac = (int)upscale, sigma0 = ps_config::sigma, L = levels:
 *         S      = L * (log2f(sigma) + up_fac - log2f(sigma0))
 *         octave = clamp(floor((S - 0.5) / L), 0, n_octaves - 1)
 *         level  = clamp(roundf(S - octave * L), 0, L + 2)        (with the explicit octave if only the level is -1)
 *     For a detected keypoint with 1 <= lpos <= L this gives back its (octave, lpos), except within float rounding of a
 *     half-integer scale.
 * n is limited only by int32 and device memory (the slot's buffers grow).  All desc_modes and norm_modes apply.
 * Detection and describe calls may alternate on one slot; a describe call launches directly, never through the slot's
 * CUDA graph, and ps_stage_ms reports 0 ms for its extrema stage.
 * Returns PS_ERR_ARG for n < 0, kps == NULL with n > 0 or unknown flags, PS_ERR_TOO_LARGE as ps_submit_*; n = 0 is valid
 * and gives zero features. */
int ps_describe_u8 (ps_ctx* ctx, int slot, const uint8_t* host_img, int w, int h, const ps_keypoint* kps, int n, int flags);
int ps_describe_f32(ps_ctx* ctx, int slot, const float*   host_img, int w, int h, const ps_keypoint* kps, int n, int flags);

/* page-locked host memory for images and results (thin wrappers of cudaHostAlloc / cudaFreeHost).
 * ps_submit_* and ps_download detect page-locked buffers and copy straight from / into them; pageable
 * buffers are staged through the slot's own pinned buffers (one extra host memcpy). */
void* ps_host_alloc(size_t bytes);
void  ps_host_free(void* p);
/* waits until the input image of the slot's last ps_submit_* has been consumed (its host -> device copy
 * is complete): after this a page-locked input buffer may be reused.  Does not wait for the kernels. */
int ps_wait_input(ps_ctx* ctx, int slot);
/* waits for the slot's stream without reading anything */
int ps_sync(ps_ctx* ctx, int slot);

/* replaces Octave::download_and_save_array (reference sift_octave.cu:111-188): one pyramid plane,
 * W*H floats, row-major, no pitch.  which = PS_PLANE_GAUSS (level 0..L+2) / PS_PLANE_DOG (0..L+1). */
int ps_debug_plane(ps_ctx* ctx, int slot, int octave, int level, int which, float* out);
/* extrema of the last image of the slot (after orientation); returns count, fills up to cap */
int ps_debug_extrema(ps_ctx* ctx, int slot, ps_extremum* out, int cap);
/* which evaluation of octave 0 / level 0 is bit-exact for a w x h input scaled to W x H with the reference's `shift`
 * and a row filter of radius R (host arithmetic only, no device needed): 0 = ideal 2x pattern, 1 = neighbouring outputs
 * share their texture fetches, 2 = every tap fetched at its own coordinate (see DESIGN.md, input texture). */
int ps_debug_level0_plan(int w, int h, int W, int H, float shift, int R);
/* geometry of the last image submitted to the slot */
int ps_slot_geometry(ps_ctx* ctx, int slot, int32_t* n_octaves, int32_t* W, int32_t* H);
/* CUDA-event time of each stage of the slot's last image (ms); enable with ps_set_timing(ctx,1) */
int ps_set_timing(ps_ctx* ctx, int enable);
int ps_stage_ms(ps_ctx* ctx, int slot, float ms[PS_NUM_STAGES]);
/* number of kernels this library launched since ps_create (all slots) */
int64_t ps_launch_count(const ps_ctx* ctx);
/* the CUDA stream (cudaStream_t) of a slot, for event timing by the caller */
void* ps_slot_stream(ps_ctx* ctx, int slot);
/* run only the pyramid stage on the slot's current input (benchmark / roofline hook) */
int ps_run_pyramid_only(ps_ctx* ctx, int slot);
/* run ONE pyramid launch on the slot's current planes (roofline hook): level 0 of octave 0 is the
 * input-image kernel, any other (octave, level >= 1) the fused blur+DoG kernel of that level */
int ps_run_level_only(ps_ctx* ctx, int slot, int octave, int level);

#ifdef __cplusplus
}
#endif
#endif /* POPSIFT_B200_H */
