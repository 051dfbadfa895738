/* TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference PopSift hot path.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load
 * this library.  The product (popsift_b200/csrc) never links to or calls it.
 *
 * Parity pin: tests/golden/ holds outputs of the UNMODIFIED reference library
 * (oracle/_ref, built from /root/reference by oracle/build_ref.sh) run on a B200;
 * tests/test_oracle_golden.py checks this restatement against them.
 */
#ifndef SIFT_ORACLE_H
#define SIFT_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_GAUSS_ALIGN  32   /* sift_constants.h:37 */
#define ORC_GAUSS_LEVELS 12   /* sift_constants.h:38 */
#define ORC_MAX_OCTAVES  20   /* sift_conf.h:12 */

/* enum values follow sift_conf.h:33-107 */
enum { ORC_MODE_POPSIFT = 0, ORC_MODE_OPENCV = 1, ORC_MODE_VLFEAT = 2 };
enum { ORC_NORM_ROOTSIFT = 0, ORC_NORM_CLASSIC = 1 };

typedef struct orc_config {
    int32_t octaves;          /* -1 = auto (popsift.cpp:118-122) */
    int32_t levels;           /* 3 */
    float   sigma;            /* 1.6 */
    float   edge_limit;       /* 10 */
    float   threshold;        /* 0.04 */
    float   upscale;          /* 1.0 (= -downsampling) */
    float   initial_blur;     /* 0.5 */
    int32_t has_initial_blur; /* 1 */
    int32_t sift_mode;        /* ORC_MODE_* */
    int32_t norm_mode;        /* ORC_NORM_* */
    int32_t norm_multi;       /* 0 */
    int32_t max_extrema;      /* 100000 */
    int32_t scaling_mode;     /* 0 = ScaleDefault, 1 = ScaleDirect (sift_conf.h; s_pyramid_build.cu:499-514) */
    int32_t gauss_direct;     /* 1 = --gauss-mode vlfeat-direct (VLFeat_Relative_All, s_pyramid_build.cu:543-546) */
    int32_t gauss_relative;   /* 1 = --gauss-mode relative / vlfeat-hw-interpolated (VLFeat_Relative, :515-542) */
    int32_t gauss_fixed;      /* 4 = --gauss-mode fixed9, 7 = fixed15 (Fixed9 / Fixed15: s_pyramid_fixed.cu), 0 = off */
} orc_config;

typedef struct orc_gauss_table {
    float   filter[ORC_GAUSS_LEVELS * ORC_GAUSS_ALIGN];
    float   sigma[ORC_GAUSS_LEVELS];
    int32_t span[ORC_GAUSS_LEVELS];
} orc_gauss_table;

/* What tex2DLayered<float> returns for the reference's UNNORMALIZED, linear, clamped float textures (the data and
 * intermediate planes, sift_octave.cu:243-252,311-325) between the texels of one row: c = the coordinate handed to the
 * texture unit (readTex has already added 0.5).  Measured with `texprobe lcoords` (tests/golden/texture_lcoords.npz). */
float orc_tex_lin1d(const float* row, int n, float c);

typedef struct orc_tables {
    orc_gauss_table inc;                 /* gauss_filter.cu:173-188 */
    float   dd_filter0[ORC_GAUSS_ALIGN]; /* dd table row 0, gauss_filter.cu:227-238 */
    float   dd_sigma0;
    int32_t dd_span0;
    float   peak_threshold;              /* sift_conf.cu:276-279 */
    float   sigma_k;                     /* sift_constants.cu:27 */
    /* all rows of the dd table (gauss_filter.cu:216-238), used by ScaleDirect */
    float   dd_filter[ORC_MAX_OCTAVES * ORC_GAUSS_ALIGN];
    float   dd_sigma[ORC_MAX_OCTAVES];
    int32_t dd_span[ORC_MAX_OCTAVES];
    orc_gauss_table abs_o0;              /* gauss_filter.cu:190-199: every level of octave 0 from the input image */
    /* the incremental rows transformed for hardware interpolation (gauss_filter.cu:372-405) */
    float   inc_ifilter[ORC_GAUSS_LEVELS * ORC_GAUSS_ALIGN];
    int32_t inc_ispan[ORC_GAUSS_LEVELS];
    orc_gauss_table abs_oN;              /* gauss_filter.cu:200-214: levels >= 1 from level 0 of the same octave */
} orc_tables;

/* same layout as popsift::Feature (features.h:23-37), 72 bytes */
typedef struct orc_feature {
    int32_t debug_octave;
    float   xpos, ypos, sigma;
    int32_t num_ori;
    float   orientation[4];
    int32_t pad_;
    int64_t desc_idx[4];   /* index into the descriptor array (-1 = none) */
} orc_feature;

typedef struct orc_ctx orc_ctx;

void     orc_default_config(orc_config* c);
int      orc_compute_tables(const orc_config* c, orc_tables* t);
/* geometry: returns number of octaves, fills W[],H[] (popsift.cpp:109-126; sift_pyramid.cu:129-134) */
int      orc_geometry(const orc_config* c, int w, int h, int32_t* W, int32_t* H);

orc_ctx* orc_create(const orc_config* c, int w, int h);
void     orc_destroy(orc_ctx* ctx);
/* stage bit mask: 1 pyramid, 2 extrema, 4 orientation, 8 descriptors */
int      orc_run_u8(orc_ctx* ctx, const uint8_t* img, int stages);
int      orc_run_f32(orc_ctx* ctx, const float* img, int stages);   /* PopSift::FloatImages */
int      orc_num_octaves(const orc_ctx* ctx);
int      orc_octave_dims(const orc_ctx* ctx, int octave, int32_t* W, int32_t* H);
const float* orc_gauss_plane(const orc_ctx* ctx, int octave, int level);
const float* orc_dog_plane(const orc_ctx* ctx, int octave, int level);
const orc_tables* orc_get_tables(const orc_ctx* ctx);
/* initial extrema (octave-local coordinates): rows of 5 floats x,y,sigma,lpos,octave */
int      orc_num_extrema(const orc_ctx* ctx);
int      orc_get_extrema(const orc_ctx* ctx, float* out5);
int      orc_counts(const orc_ctx* ctx, int32_t* n_feat, int32_t* n_desc);
int      orc_download(const orc_ctx* ctx, orc_feature* feat, float* desc128);
/* descriptors of n caller-given keypoints: kp4 = n x {x, y, sigma, angle} (octave-local), oct_lpos = n x {octave, lpos} */
int      orc_describe(const orc_ctx* ctx, int n, const float* kp4, const int32_t* oct_lpos, float* desc128);
/* stand-alone: normalised value the input texture returns (pins the texture model) */
float    orc_tex_u8(const uint8_t* img, int w, int h, float rx, float ry);
float    orc_tex_f32(const float* img, int w, int h, float rx, float ry);
int      orc_set_threads(int n);

#ifdef __cplusplus
}
#endif
#endif
