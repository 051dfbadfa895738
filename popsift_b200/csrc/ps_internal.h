// Internal (device + host) structures shared by the kernels and the C-ABI layer.
#pragma once
#include "popsift_b200.h"
#include "popsift_b200_pose.h"
#include "popsift_b200_tracks.h"
#include "popsift_b200_triangulate.h"
#include "popsift_b200_bundle.h"
#include "popsift_b200_global.h"
#include "popsift_b200_viewgraph.h"
#include "popsift_b200_twoview.h"
#include "popsift_b200_depth.h"
#include "popsift_b200_mesh.h"
#include "popsift_b200_render.h"

#include <cuda_runtime.h>
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

namespace psb {

constexpr int kMaxOctaves = PS_MAX_OCTAVES;
constexpr int kMaxPlanes  = PS_GAUSS_LEVELS + 3;   // L+3 <= 15
constexpr int kOriBins    = 36;                    // reference sift_constants.h:41
constexpr int kMaxLevels  = PS_GAUSS_LEVELS;

// A candidate from the DoG scan (reference InitialExtremum, sift_extremum.h:25-39, without
// the grid-filter fields).
struct InitialExtremum {
    float xpos, ypos;
    int   lpos;
    float sigma;
};

// Per-image device counters (reference ExtremaCounters, sift_pyramid.h:21-35).
struct Counters {
    int ext_ct[kMaxOctaves];   // extrema found per octave (may exceed max_extrema; clamp on use)
    int ext_total;             // after clamping, written by the orientation-prefix kernel
    int ori_total;
    int overflow;              // bit 0: extrema capacity hit, bit 1: descriptor capacity hit
    int work_ori;              // work-stealing cursors
    int work_desc;
    int filtered;              // the grid filter fired: the orientation stage reads ext_ct_f / the filtered array
    int ext_ct_f[kMaxOctaves]; // extrema per octave that survived the grid filter
    int ori_needed;            // descriptors the image has (may exceed desc_capacity: the host then grows the buffers)
    int pad_[1];
};

// grid filter (k_filter.cu; reference s_filtergrid.cu:112-325)
struct FilterCfg { int max_extrema, grid, sort; };
struct FilterPlan {
    int active, limit, total, pad_;
    int cell_count[PS_MAX_FILTER_GRID * PS_MAX_FILTER_GRID];
};

// One octave's planes in HBM: linear float32, row pitch a multiple of 32 floats (128 B).
struct OctaveView {
    float* gauss;       // (levels+3) planes, plane stride = plane
    // (levels+2) planes, DoG[l] = G[l+1] - G[l].  Written only on request (ps_debug_plane -> launch_dog_planes): during an
    // extraction nothing writes or reads this region; the extrema stage forms every DoG sample it needs from the two
    // Gaussian planes with the same __fsub_rn, so the region may hold anything (e.g. an earlier image's planes).
    float* dog;
    // candidate lists of the `levels` scanned DoG planes (see CandSink): level q (DoG plane q+1), block b of
    // the level kernel owns entries [(q*cand_blocks + b) * cand_region, +cand_cnt[q*cand_blocks + b])
    uint32_t* cand;
    int*   cand_cnt;
    int    cand_blocks, cand_region;
    int    w, h;
    int    pitch;       // floats per row
    size_t plane;       // floats per plane = pitch * h
};

// Kernel-visible description of one slot's pyramid.
struct PyramidView {
    OctaveView oct[kMaxOctaves];
    int        num_octaves;
    int        levels;      // L
    int        cands_filled;   // the pyramid kernels appended the candidate lists of this image
    // the block counts of all octaves (oct[o].cand_cnt, contiguous in octave order), their number and the
    // array their exclusive prefix sum is written to (cand_regions + 1 entries)
    int*       cand_cnt_all;
    int*       cand_prefix;
    int        cand_regions;
};

// Where a pyramid kernel reports the DoG pixel pairs (x even) in which a sample passes the peak
// threshold while it writes Gaussian level l (DoG[l-1] = G[l] - G[l-1] in registers): the extrema stage then only visits those (a few per thousand
// pixels) instead of scanning every plane again.  Each block of the kernel owns a private region of the
// list and a count (zeroed per image), so the kernel needs a shared-memory counter but no global atomic.
struct CandSink {
    uint32_t* list;     // blocks x region entries: x | y << 16 of the pair's left pixel
    int*      counts;   // blocks
    float     thr;
    int       region;   // entries per block
};

// Small constants consumed by the extrema / orientation / descriptor kernels
// (reference ConstInfo, sift_constants.h:56-67).
struct Consts {
    float sigma0;
    float sigma_k;
    float edge_limit;
    float threshold;        // peak threshold
    int   max_extrema;      // per octave
    int   ext_capacity;     // total Extremum records per slot
    int   desc_capacity;    // total descriptors per slot
    int   norm_multi;
    int   norm_mode;
    int   sift_mode;
    int   up_fac;           // int(upscale), reference sift_pyramid.cu:297
};

// |DoG| below this can never be an extremum (reference s_extrema.cu:425-440: the three modes' pre-test)
#ifdef __CUDACC__
__host__ __device__
#endif
inline float extrema_threshold(const Consts& k)
{
    // float(0.8) * 2 == float(1.6): the VLFeat and PopSift expressions agree bit for bit
    return k.sift_mode == PS_MODE_OPENCV ? floorf(k.threshold) : 1.6f * k.threshold;
}

// the calling thread's message for ps_last_error(NULL); the stateless entry points (ps_batch.cu) report through it
void set_last_error(const std::string& msg);

// multiprocessors of the CURRENT device (cudaDeviceProp::multiProcessorCount, cached per device; 132 on H100 SXM):
// every fixed grid and the one-wave partition of the pyramid kernels are sized from it
int sm_count();

// ---- launchers (defined in the k_*.cu files); all asynchronous on `st`, return #kernels launched

struct GaussRow { float tap[PS_GAUSS_ALIGN]; int span; };

int level0_plan_for(int w, int h, int W, int H, float shift, int R);   // k_pyramid.cu: LEVEL0_* choice for one geometry
// octave 0, level 0 from the 8-bit or float input image
// (octave > 0: Config::ScaleDirect, the same pass onto a smaller octave with that octave's dd row and shift 0.5)
int launch_level0_u8(const uint8_t* img, size_t img_pitch, int w, int h, float upscale, int sift_mode,
                     const OctaveView& o0, const GaussRow& dd, const GaussRow& inc0, cudaStream_t st, int octave = 0);
// levels 0 and 1 of octave 0 in one launch where the fused kernel applies (8-bit input up-scaled exactly 2x, both radii 5,
// marching kernels); 0 (nothing launched) anywhere else
int launch_level01_u8(const uint8_t* img, size_t img_pitch, int w, int h, float upscale, int sift_mode,
                      const OctaveView& o0, const GaussRow& dd, const GaussRow& inc0, const GaussRow& g1, cudaStream_t st);
int launch_level0_f32(const float* img, size_t img_pitch_floats, int w, int h, float upscale, int sift_mode,
                      const OctaveView& o0, const GaussRow& dd, const GaussRow& inc0, cudaStream_t st, int octave = 0);
// --gauss-mode vlfeat-direct (VLFeat_Relative_All): one level of octave 0 straight from the input image; the next
// octave's level 0 then comes from its own small kernel
int launch_level0_abs_u8(const uint8_t* img, size_t img_pitch, int w, int h, float upscale, int sift_mode,
                         const OctaveView& o0, int level, const GaussRow& taps, cudaStream_t st);
int launch_level0_abs_f32(const float* img, size_t img_pitch_floats, int w, int h, float upscale, int sift_mode,
                          const OctaveView& o0, int level, const GaussRow& taps, cudaStream_t st);
// DoG planes 0 .. nplanes-1 of one octave from its Gaussian planes (on request only: see OctaveView::dog)
int launch_dog_planes(const OctaveView& o, int nplanes, cudaStream_t st);
// --gauss-mode relative (VLFeat_Relative): the first horizontal pass alone, and one interpolated pass over a plane
int launch_level0_rows_u8(const uint8_t* img, size_t img_pitch, int w, int h, float upscale, int sift_mode,
                          const OctaveView& o0, float* dst, const GaussRow& dd, cudaStream_t st, int octave = 0);
int launch_level0_rows_f32(const float* img, size_t img_pitch_floats, int w, int h, float upscale, int sift_mode,
                           const OctaveView& o0, float* dst, const GaussRow& dd, cudaStream_t st, int octave = 0);
// --gauss-mode fixed9 / fixed15 (s_pyramid_fixed.cu): one level of octave 0 from the input image / of an octave >= 1 from its level 0
int launch_fixed_level0_u8(const uint8_t* img, size_t img_pitch, int w, int h, float upscale, const OctaveView& o0, int level,
                           const GaussRow& taps, int S, float* scratch, cudaStream_t st);
int launch_fixed_level0_f32(const float* img, size_t img_pitch_floats, int w, int h, float upscale, const OctaveView& o0, int level,
                            const GaussRow& taps, int S, float* scratch, cudaStream_t st);
int launch_fixed_levelN(const OctaveView& o, int level, const GaussRow& taps, int S, float* scratch, cudaStream_t st);
int launch_interp_pass(const float* src, float* dst, int W, int H, int pitch, const GaussRow& f, int ispan, int along_x, cudaStream_t st);
int launch_decimate(const OctaveView& prev, int level, const OctaveView& next, cudaStream_t st);
// level l >= 1 of one octave: blur level l-1 -> level l (no DoG plane is written); if next0 != nullptr
// also writes every second pixel into the next octave's level 0.
// `sink` (optional) receives the threshold-passing samples of the DoG plane; only honoured when
// blur_level_collects(g) is true.
int launch_blur_level(const OctaveView& o, int level, const GaussRow& g, const OctaveView* next, const CandSink* sink,
                      cudaStream_t st);
bool blur_level_collects(const GaussRow& g);
// layout of the candidate lists of one w x h plane (k_partition.h): blocks, entries per block, and a
// monotonic upper bound of blocks * entries (memory budget)
int cand_blocks_for(int w, int h);
int cand_region_for(int w, int h);
long long cand_entry_bound_for(int w, int h);

int launch_find_extrema(const PyramidView& pyr, const Consts& k, InitialExtremum* iext, Counters* ct, cudaStream_t st);
// grid filter between the extrema and the orientation stage; no-op (returns 0) when fc.max_extrema <= 0.
// keep: one byte per initial extremum (num_octaves * max_extrema); iext_f: a second InitialExtremum array
int launch_grid_filter(const PyramidView& pyr, const Consts& k, const FilterCfg& fc, const InitialExtremum* iext,
                       InitialExtremum* iext_f, unsigned char* keep, size_t keep_bytes, FilterPlan* plan, Counters* ct,
                       cudaStream_t st);
// slice_sum: ext_capacity / PS_ORI_SLICE + 1 ints, zeroed per image
#define PS_ORI_SLICE 256
// iext_f: the grid-filtered extrema (read instead of iext when ct->filtered); may be nullptr when the filter is off
int launch_orientation(const PyramidView& pyr, const Consts& k, const InitialExtremum* iext, const InitialExtremum* iext_f, ps_extremum* ext,
                       int* feat_to_ext, int* slice_sum, Counters* ct, cudaStream_t st);
// the two halves of launch_orientation: the orientation kernel alone (writes ext[] in octave order and adds each record's
// num_ori to slice_sum), and the exclusive scan of ext[].num_ori over the first ext_total records (idx_ori, feat_to_ext,
// ext_total, ori_total, overflow flags), where ext_total comes from ct's per-octave counts like in the orientation kernel
int launch_orientation_only(const PyramidView& pyr, const Consts& k, const InitialExtremum* iext, const InitialExtremum* iext_f, ps_extremum* ext,
                            int* slice_sum, Counters* ct, cudaStream_t st);
int launch_ori_scatter(int num_octaves, const Consts& k, ps_extremum* ext, int* feat_to_ext, const int* slice_sum, Counters* ct, cudaStream_t st);
int launch_descriptors(const PyramidView& pyr, const Consts& k, const ps_extremum* ext, const int* feat_to_ext,
                       ps_descriptor* desc, Counters* ct, cudaStream_t st);

// describe path (k_describe.cu): caller-supplied keypoints instead of detected extrema.
// kp_ingest: validates keypoint i, picks its octave and level and writes its octave-local record.  orient = false: ext[i]
// (num_ori 1, the given angle) and its num_ori into slice_sum; orient = true: the valid keypoints are appended to the
// per-octave regions iext[o * stride ..] (count in ct_ori->ext_ct[o], source index in src[]) and only rejected ones get
// their ext[i].  Either way ct->ext_ct[0] = n, so that launch_ori_scatter with max_extrema >= n scans ext[0, n).
int launch_kp_ingest(const PyramidView& pyr, const Consts& k, const ps_keypoint* kp, int n, bool orient, ps_extremum* ext,
                     InitialExtremum* iext, int* src, int stride, int* slice_sum, Counters* ct_ori, Counters* ct, cudaStream_t st);
// the orientation kernel's records (octave order, ext_sorted) back to input order in ext, with their num_ori into slice_sum
int launch_kp_restore(int num_octaves, const ps_extremum* ext_sorted, const int* src, int stride, int n, ps_extremum* ext,
                      int* slice_sum, const Counters* ct_ori, cudaStream_t st);
// Feature i gets keypoint i's own x, y and sigma bits
int launch_kp_finish(const ps_keypoint* kp, int n, ps_feature* feat, cudaStream_t st);
// --desc-mode grid / igrid / iloop / notile (k_desc_modes.cu; reference s_desc_grid.cu, s_desc_igrid.cu, s_desc_iloop.cu,
// s_desc_notile.cu); PS_DESC_LOOP goes through launch_descriptors
int launch_descriptors_mode(int mode, const PyramidView& pyr, const Consts& k, const ps_extremum* ext, const int* feat_to_ext,
                            ps_descriptor* desc, Counters* ct, cudaStream_t st);
int launch_prep_features(const Consts& k, const ps_extremum* ext, ps_feature* feat, const Counters* ct, cudaStream_t st);
// device copy of the Feature records: desc[] become pointers into `desc` (first index is in pad_)
int launch_fix_feature_pointers(ps_feature* feat, ps_descriptor* desc, int n, cudaStream_t st);

// brute-force 2-NN matcher (k_match.cu; reference features.cu:165-304): out = n_left x (best, second, accept), device
// memory; asynchronous on `st`; returns the number of kernels launched or -1 (*err set)
int run_match(const ps_descriptor* l, int nl, const ps_descriptor* r, int nr, int32_t* out, int flags, cudaStream_t st, const char** err);
// many pairs (indices into sets / n_desc, already validated): pair p's rows start at row sum_{q<p} n_desc[pairs[2q]] of out.
// EXACT runs match_exact_kernel pair by pair; AUTO / TENSOR plan groups of pairs (k_match_plan.h) and run one split, one
// tensor-core and one re-rank launch per group
int run_match_batch(const ps_descriptor* const* sets, const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs,
                    int32_t* out, int flags, cudaStream_t st, const char** err);
// bytes one group of the batched matcher may use (POPSIFT_B200_MATCH_WS, default 1 GB)
size_t match_workspace_cap();
// flags after the POPSIFT_B200_MATCH=exact|tc override (k_match.cu)
int match_choice(int flags);

// 8-bit descriptors (k_match_u8.cu): out[i] = roundf(min(max(in[i], 0), 255)) (NaN -> 0) for n x 128 components
int run_descriptors_to_u8(const ps_descriptor* in, int n, uint8_t* out, cudaStream_t st);
// run_match_batch for sets of n_desc[i] x 128 uint8_t (16-byte aligned): same pair list, same output rows, exact integer
// distances.  EXACT runs match_u8_exact_kernel pair by pair; AUTO / TENSOR plan groups of pairs with 132-byte rows and run
// one pack, one integer tensor-core and one finalize launch per group
int run_match_u8_batch(const uint8_t* const* sets, const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs,
                       int32_t* out, int flags, cudaStream_t st, const char** err);

// geometric verification (k_verify.cu), arguments already validated.  Correspondences of matched pairs: one gather launch;
// n_corr (host) is written before the call returns.  Returns the number of kernels launched or -1 (*err set).
int run_match_correspondences(const ps_feature* const* feat, const int32_t* const* rev, const int32_t* n_desc, const int32_t* pairs,
                              int n_pairs, const int32_t* match, float* corr, int32_t* src, int32_t* n_corr, cudaStream_t st,
                              const char** err);
// batched RANSAC (normalise, solve, score, select / refit, taps); asynchronous on `st`
int run_verify_batch(int n_pairs, const float* corr, const int32_t* corr_start, const int32_t* n_corr, const ps_verify_params& prm,
                     float* d_models, int32_t* d_n, uint8_t* d_mask, const ps_verify_taps* taps, cudaStream_t st, const char** err);
// calibrated two-view geometry (include/popsift_b200_pose.h, k_pose.cu), arguments already validated: calibrate, solve,
// compact, score, select / pose, taps.  Synchronises `st` once, to plan the scoring on each pair's valid hypotheses.
int run_relative_pose_batch(int n_pairs, const float* corr, const int32_t* corr_start, const int32_t* n_corr, const ps_camera* cams,
                            const ps_pose_params& prm, ps_two_view* d_out, uint8_t* d_mask, float* d_points, const ps_verify_taps* taps,
                            cudaStream_t st, const char** err);

// guided matching (include/popsift_b200_guided.h), arguments already validated: run_match_batch / run_match_u8_batch with
// right descriptor j of pair p eligible for left descriptor i only when their keypoints pass the test of k_guided.h under
// the pair's model (models: DEVICE, 9 floats per pair; model: PS_GEOM_*; threshold in pixels).  EXACT runs the CUDA-core
// guided kernels pair by pair; AUTO / TENSOR plan with rows 8 bytes larger (the pixel position) and run one split / pack,
// one position, one guided tensor-core and one re-rank / finalize launch per group.
int run_match_guided_batch(const ps_descriptor* const* sets, const ps_feature* const* feat, const int32_t* const* rev,
                           const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs, const float* models, int model,
                           float threshold, int32_t* out, int flags, cudaStream_t st, const char** err);
int run_match_u8_guided_batch(const uint8_t* const* sets, const ps_feature* const* feat, const int32_t* const* rev,
                              const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs, const float* models, int model,
                              float threshold, int32_t* out, int flags, cudaStream_t st, const char** err);

// image retrieval (include/popsift_b200_retrieval.h, k_retrieval.cu), arguments already validated; asynchronous on `st`,
// return the number of kernels launched or -1 (*err set).  Assignment is run_match_batch against the centroids.
int run_vlad_train(const ps_descriptor* const* sets, const int32_t* n_desc, int n_sets, int k, int iters, uint64_t seed,
                   float* centroids, int flags, cudaStream_t st, const char** err);
int run_vlad_encode(const ps_descriptor* const* sets, const int32_t* n_desc, int n_sets, int k, const float* centroids,
                    float* vlad, int32_t* assign, int flags, cudaStream_t st, const char** err);
int run_retrieve_pairs(int n, const float* vec, int dim, int m, int32_t* nbr, float* score, cudaStream_t st, const char** err);

// feature tracks (include/popsift_b200_tracks.h, k_tracks.cu), arguments already validated except the edges' endpoints:
// an endpoint outside its range sets *bad_edge, and the call returns before writing any output.  Synchronous on `st` (the
// flag and the counts are read back); return the number of kernels launched or -1 (*err set).
// One pair of ps_tracks_from_matches: first is filled in by the run.
struct TrackPair {
    long long first;                  // the pair's first correspondence in the concatenation of all pairs' correspondences
    long long row0;                   // its first row of d_match / d_src / d_inlier_mask
    const int32_t* rev_l;
    const int32_t* rev_r;
    int32_t off_l, off_r;             // global id of feature 0 of the left / right set
    int32_t n_l, n_r;                 // descriptors
    int32_t nf_l, nf_r;               // features
    int32_t n_corr, pad_;
};
int run_tracks_from_edges(int n_sets, const int32_t* n_feat, int n_edges, const int32_t* edges, int min_length, int32_t* track_of,
                          int32_t* track_start, int32_t* members, ps_track_counts* counts, bool* bad_edge, cudaStream_t st,
                          const char** err);
int run_tracks_from_matches(int n_sets, const int32_t* n_feat, const std::vector<TrackPair>& pairs, const int32_t* match,
                            const int32_t* src, const uint8_t* mask, int min_length, int32_t* track_of, int32_t* track_start,
                            int32_t* members, ps_track_counts* counts, bool* bad_edge, cudaStream_t st, const char** err);

// multi-view triangulation (include/popsift_b200_triangulate.h, k_triangulate.cu), arguments already validated except the
// member ids and d_track_start, which the ray pass checks: a bad one sets *bad, and the call returns before writing any
// output.  Synchronous on `st` (the flag and the counts are read back); returns the number of kernels launched or -1.
int run_triangulate_tracks(int n_sets, const int32_t* n_feat, const ps_feature* const* feat, const ps_camera* cams, const ps_rigid* poses,
                           int n_tracks, const int32_t* track_start, const int32_t* members, int n_members,
                           const ps_triangulate_params& prm, ps_track_point* points, uint8_t* obs_mask, float* obs_error,
                           ps_triangulate_counts* counts, bool* bad, cudaStream_t st, const char** err);

// bundle adjustment (include/popsift_b200_bundle.h, k_bundle.cu), arguments already validated except the member ids and
// d_track_start, which the first pass checks: a bad one sets *bad, and the call returns before writing any output.
// Synchronous on `st` (one small read-back per LM iteration); *report and poses_out are written when it returns >= 0 with
// *bad false.  Returns the number of kernels launched or -1 (*err set).
int run_bundle_adjust(int n_sets, const int32_t* n_feat, const ps_feature* const* feat, const ps_camera* cams, const ps_rigid* poses_in,
                      int n_tracks, const int32_t* track_start, const int32_t* members, int n_members, ps_track_point* points,
                      const uint8_t* obs_mask, const uint8_t* fixed, const ps_bundle_params& prm, ps_rigid* poses_out, float* obs_error,
                      ps_bundle_report* report, bool* bad, cudaStream_t st, const char** err);

// global poses (include/popsift_b200_global.h, k_global.cu), arguments already validated.  Rotation averaging reads the
// two-view records back once, starts on the host and writes every output when it returns >= 0.  Positioning: the member
// ids and d_track_start are checked by the first pass (a bad one sets *bad, and the call returns before writing any
// output); otherwise every output is written.  Synchronous on `st`; return the number of kernels launched or -1 (*err set).
int run_rotation_averaging(int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view, const ps_rotation_params& prm,
                           double* R_out, uint8_t* registered, float* pair_error, ps_rotation_report* report, cudaStream_t st,
                           const char** err);
int run_global_positioning(int n_sets, const int32_t* n_feat, const ps_feature* const* feat, const ps_camera* cams, const double* R,
                           const uint8_t* registered, int n_tracks, const int32_t* track_start, const int32_t* members, int n_members,
                           const ps_position_params& prm, ps_rigid* poses_out, uint8_t* positioned, double* X_out,
                           ps_position_report* report, bool* bad, cudaStream_t st, const char** err);

// view-graph filter (include/popsift_b200_viewgraph.h, k_viewgraph.cu), arguments already validated (duplicates included)
// and n_pairs > 0.  Synchronous on `st`; keep, stats (optional), d_kept (optional) and *report are written when it returns
// >= 0.  Returns the number of kernels launched or -1 (*err set).
int run_view_graph_filter(int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view, const ps_view_graph_params& prm,
                          uint8_t* keep, ps_cycle_stats* stats, ps_two_view* d_kept, ps_view_graph_report* report, cudaStream_t st,
                          const char** err);

// two-view configuration (include/popsift_b200_twoview.h, k_twoview.cu), arguments already validated and n_pairs > 0.
// Synchronous on `st`; info is written when it returns >= 0.  Returns the number of kernels launched or -1 (*err set).
int run_two_view_config_batch(int n_pairs, const float* corr, const int32_t* corr_start, const int32_t* n_corr, const ps_camera* cams,
                              const ps_two_view* d_essential, const uint8_t* d_essential_mask, const int32_t* d_f_inliers,
                              const float* d_homography, const uint8_t* d_h_mask, const ps_two_view_config_params& prm,
                              ps_two_view* d_out, uint8_t* d_out_mask, float* d_points, ps_two_view_info* info, cudaStream_t st,
                              const char** err);

// dense depth maps and their consistency filter (include/popsift_b200_depth.h, k_depth.cu), arguments already validated
// and n_refs > 0.  Synchronous on `st`; the report is written when they return >= 0.  Return the number of kernels
// launched or -1 (*err set).
int run_depth_maps(int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs, const int32_t* refs,
                   const float* ranges, const int32_t* src_start, const int32_t* src_sets, const ps_depth_params& prm,
                   float* const* d_depth, float* const* d_cost, uint8_t* const* d_n_src, ps_depth_report* report, cudaStream_t st,
                   const char** err);
int run_depth_filter(int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs, const int32_t* refs,
                     const int32_t* src_start, const int32_t* src_sets, const float* const* d_depth, const ps_depth_filter_params& prm,
                     uint8_t* const* d_n_consistent, ps_dense_point* d_points, ps_depth_filter_report* report, cudaStream_t st,
                     const char** err);

// surface meshes (include/popsift_b200_mesh.h, k_mesh.cu), arguments already validated.  Asynchronous clear; the other two
// are synchronous on `st`: the integration writes *report when it returns >= 0 and n_views > 0; the extraction writes
// *report when it returns >= 0, and the outputs only when *overflow is false.  Return the number of kernels launched or
// -1 (*err set).
int run_volume_clear(const ps_volume& vol, cudaStream_t st, const char** err);
int run_tsdf_integrate(int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, const float* const* d_depth,
                       const uint8_t* const* d_n_consistent, const ps_tsdf_params& prm, const ps_volume& vol, ps_tsdf_report* report,
                       cudaStream_t st, const char** err);
int run_tsdf_mesh(const ps_volume& vol, const ps_mesh_params& prm, int64_t max_vertices, int64_t max_triangles, ps_mesh_vertex* d_vertices,
                  int32_t* d_triangles, ps_mesh_report* report, bool* overflow, cudaStream_t st, const char** err);

// mesh rendering and texturing (include/popsift_b200_render.h, k_render.cu), arguments already validated except the
// vertex indices, which a first kernel checks: a bad one sets *bad, and the call returns before writing any output.
// Render needs n_views > 0, texture n_triangles > 0.  Synchronous on `st`; *report is written when they return >= 0 with
// *bad false.  Return the number of kernels launched or -1 (*err set).
int run_mesh_render(int n_views, const int32_t* sizes, const ps_camera* cams, const ps_rigid* poses, const ps_mesh_vertex* d_vertices,
                    int64_t n_vertices, const int32_t* d_triangles, int64_t n_triangles, const ps_render_params& prm, float* const* d_depth,
                    int32_t* const* d_tri, ps_render_report* report, bool* bad, cudaStream_t st, const char** err);
int run_mesh_texture(int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, const float* const* d_depth,
                     const ps_mesh_vertex* d_vertices, int64_t n_vertices, const int32_t* d_triangles, int64_t n_triangles,
                     const ps_texture_params& prm, uint8_t* d_atlas, int32_t* d_view, ps_texture_report* report, bool* bad,
                     cudaStream_t st, const char** err);

} // namespace psb
