/* Mesh rendering and texturing (an addition to the reference's interface): a triangle mesh rendered into posed views with
 * a z-buffer, and a texture atlas sampled from the grey images, one view per triangle chosen by visibility.
 *
 * ps_tsdf_mesh ends with a mesh whose only appearance is the per-vertex grey of the volume, a running mean at voxel
 * resolution.  The last step of every photogrammetry pipeline is texturing: AliceVision's Texturing node follows Meshing,
 * OpenMVS follows ReconstructMesh with TextureMesh.  Both rest on one primitive: rendering the mesh into a posed view with
 * a z-buffer, which tells which views see a triangle and what depth a view sees.  The rendered maps are in ps_depth_maps'
 * layout (camera-frame z, row stride width), so they can feed ps_depth_filter or ps_tsdf_integrate as they are.
 * Everything is deterministic: the z-buffer is a 64-bit atomicMin on (depth bits, triangle), and no floating-point atomic
 * is used anywhere.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_RENDER_H
#define POPSIFT_B200_RENDER_H

#include "popsift_b200_mesh.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_render_params {         /* 8 bytes */
    float   z_near;                       /* near plane, camera-frame z, finite and > 0                                */
    int32_t pad_;                         /* ignored                                                                   */
} ps_render_params;

typedef struct ps_render_report {         /* 24 bytes, HOST */
    int64_t n_drawn;                      /* (triangle, view) pairs rasterised: steps 1 and 2 passed, box not empty    */
    int64_t n_big;                        /* of those, the pairs whose box has more than kBigTri pixels (k_render.cu)  */
    int64_t n_covered;                    /* pixels, over all views, with a triangle                                   */
} ps_render_report;

typedef struct ps_texture_params {        /* 24 bytes */
    int32_t cell;                         /* texels per cell side, 3 .. 64                                             */
    int32_t cells_per_row;                /* >= 1; atlas width = cells_per_row cell <= 65535                           */
    float   depth_tol;                    /* relative occlusion tolerance, finite and >= 0                             */
    float   min_cos;                      /* facing test, [0, 1)                                                       */
    float   z_near;                       /* as ps_render_params                                                       */
    int32_t pad_;                         /* ignored                                                                   */
} ps_texture_params;

typedef struct ps_texture_report {        /* 16 bytes, HOST */
    int64_t n_viewed;                     /* triangles with a view                                                     */
    int64_t n_fallback;                   /* triangles textured from the vertex grey                                   */
} ps_texture_report;

/* Renders triangles d_triangles[3 m .. 3 m + 2] (DEVICE int32 vertex indices) of the vertices d_vertices (DEVICE) into
 * views v = 0 .. n_views - 1 of sizes[2 v] x sizes[2 v + 1] pixels (HOST), camera cams[v] and world-to-camera pose
 * poses[v].  For each view and each triangle m with vertices V0, V1, V2 (float positions taken as double):
 *   1. Projection, as ps_tsdf_integrate steps 1-2: X_c = R V + t in double, each row ((R_r0 X + R_r1 Y) + R_r2 Z) + t_r;
 *      p = ((fx x) / z + cx, (fy y) / z + cy).  The triangle is drawn in v only when all three X_c are finite with
 *      z >= z_near and all three p are finite.  There is no near-plane clipping: a triangle that crosses the near plane is
 *      dropped whole.
 *   2. Area: with E(a, b; x, y) = (b_x - a_x)(y - a_y) - (b_y - a_y)(x - a_x), A = E(p0, p1; p2).  The triangle is drawn
 *      only when A is finite and != 0.
 *   3. Coverage: pixel (x, y) is the point (x, y), the convention of the Feature records and ps_camera.  The candidates
 *      are the pixels of the box ceil(min p_x) .. floor(max p_x), ceil(min p_y) .. floor(max p_y) clamped to the image.
 *      With E0 = E(p1, p2; x, y), E1 = E(p2, p0; x, y), E2 = E(p0, p1; x, y), a candidate is covered when s E_i >= 0 for
 *      i = 0, 1, 2, s the sign of A.  Pixels on a shared edge are covered by both triangles and the z-buffer settles them,
 *      so there is no top-left rule and a closed mesh renders without cracks.
 *   4. Depth, perspective-correct: lambda_i = E_i / A; z = (float) (1 / ((lambda0 / z0 + lambda1 / z1) + lambda2 / z2)),
 *      in double before the rounding.  Both faces are drawn: occlusion needs both.
 *   5. Winner per pixel: the lexicographically smallest (z, m), as the 64-bit key (float bits of z) << 32 | m.
 *      d_depth[v] (float) = z, or 0 where no triangle covers the pixel; d_tri[v] (int32) = m, or -1.  Both are w x h,
 *      row stride w (HOST arrays of DEVICE pointers).
 *   6. Two identical calls give identical bytes, whatever the schedule.
 * *report: the pairs drawn, those of them rasterised by the big-triangle kernel, and the covered pixels.
 * Errors: PS_ERR_ARG before any device work, with every output and *report untouched, for: n_views, n_vertices or
 * n_triangles < 0, n_triangles >= 2^31; NULL prm or report, or (n_views > 0) NULL sizes, cams, poses, d_depth or d_tri, or
 * (n_triangles > 0) NULL d_vertices or d_triangles; a width or height outside 1 .. 65535; a camera or pose
 * ps_triangulate_tracks refuses; an output, d_vertices or d_triangles that is not device memory on `device`; z_near not
 * finite or <= 0.  A vertex index outside [0, n_vertices) is found on the device: a flag is read back before any output
 * is written, and the call returns PS_ERR_ARG with the outputs untouched.  n_views = 0 is valid (nothing is written, the
 * report is zero); n_triangles = 0 writes empty maps.  Synchronous.
 * Workspace: 8 bytes per pixel (the z-buffer keys), 144 per view, and 8 per (triangle, view) of one pass for the
 * big-triangle list; a pass covers max(1, 2^24 / n_triangles) views. */
int ps_mesh_render(int device, int n_views, const int32_t* sizes, const ps_camera* cams, const ps_rigid* poses,
                   const ps_mesh_vertex* d_vertices, int64_t n_vertices, const int32_t* d_triangles, int64_t n_triangles,
                   const ps_render_params* prm, float* const* d_depth, int32_t* const* d_tri, ps_render_report* report);

/* A texture atlas of the mesh from the grey images (HOST array of structs whose data is DEVICE memory), with d_depth[v]
 * (HOST array of DEVICE pointers) the maps ps_mesh_render gives for the same mesh and views, or any maps in that layout
 * (w x h floats of images[v]'s size, 0 = empty).  In double:
 *   1. Per triangle m: centroid C = ((V0 + V1) + V2) / 3 and normal n = (V1 - V0) x (V2 - V0), which points towards the
 *      cameras as ps_tsdf_mesh orients it.
 *   2. View v is a candidate when both tests pass:
 *      - facing: with c_v = -R^T t and d = c_v - C, n.d > 0 and n.d >= (min_cos |n|) |d| (dot products summed x, y, z);
 *      - visibility: each of the four probes V0, V1, V2, C projects as in ps_mesh_render step 1 (finite, z >= z_near),
 *        its nearest pixel q = floor(p + 1/2) lies inside the image, and it is not occluded: D = d_depth_v(q) > 0 with
 *        z > D (1 + depth_tol) is occluded.
 *   3. Score = |A_v| / 2, the projected area in pixels (ps_mesh_render step 2).  d_view[m] = the candidate with the largest
 *      score, ties to the lowest v; -1 when there is none.
 *   4. Atlas layout, a closed form: triangle m owns the cell (m mod cells_per_row, m div cells_per_row) of cell x cell
 *      texels.  The atlas is W = cells_per_row cell texels wide and H = ceil(n_triangles / cells_per_row) cell rows high,
 *      pitch W.  With a margin of b = 1 texel, the triangle's corners sit at the cell-local positions P0 = (b, b),
 *      P1 = (cell - b, b), P2 = (b, cell - b): texel-space coordinates, texel (i, j) covering [i, i + 1) x [j, j + 1).
 *   5. Texel (i, j) of a cell has its centre at (i + 1/2, j + 1/2): u = (i + 1/2 - b) / (cell - 2b), v likewise with j.
 *      (u, v) is clamped to the nearest point of the triangle u >= 0, v >= 0, u + v <= 1, in this order: u = max(u, 0),
 *      v = max(v, 0); when u + v > 1, u = clamp(((u - v) + 1) / 2, 0, 1) and v = 1 - u.  That is the Euclidean nearest
 *      point in texel space too, as P1 - P0 and P2 - P0 are orthogonal and of equal length.  beta = ((1 - u) - v, u, v).
 *      Every texel of the cell, margin and far half included, so holds the value of the triangle's nearest point: bilinear
 *      look-ups and mip-maps in a viewer do not bleed across cells.
 *   6. Texel value, with X = (beta0 V0 + beta1 V1) + beta2 V2 per coordinate:
 *      - with a view: X projects into v as in step 1; the projection is clamped to [0, w - 1] x [0, h - 1] and sampled
 *        bilinearly with ps_depth_maps step 3's rule: u0 = min(floor(u), w - 2), v0 = min(floor(v), h - 2), a = u - u0,
 *        c = v - v0, S = (1 - c) ((1 - a) I(u0, v0) + a I(u0 + 1, v0)) + c ((1 - a) I(u0, v0 + 1) + a I(u0 + 1, v0 + 1));
 *      - without a view (the fallback): S = (beta0 g0 + beta1 g1) + beta2 g2, the vertices' ps_mesh_vertex.grey.
 *      The texel is floor(S + 1/2) clamped to 0 .. 255 (NaN gives 0).  Texels of cells past the last triangle are 0, so
 *      the atlas is always complete.
 *   7. Outputs: d_atlas (uint8, W x H) and d_view (int32, n_triangles).  *report: the triangles with a view and those on
 *      the fallback.  Deterministic; two identical calls give identical bytes.
 * The caller computes the texture coordinates from step 4; no device output holds them.
 * Errors: PS_ERR_ARG before any device work, with every output and *report untouched, for: n_views, n_vertices or
 * n_triangles < 0, n_triangles >= 2^31; NULL prm or report, or (n_views > 0) NULL images, cams, poses or d_depth, or
 * (n_triangles > 0) NULL d_vertices, d_triangles, d_atlas or d_view; an image whose width or height is outside 2 .. 65535
 * or whose pitch is < width; a camera or pose ps_triangulate_tracks refuses; an image, map, d_vertices, d_triangles,
 * d_atlas or d_view that is not device memory on `device`; cell outside 3 .. 64, cells_per_row < 1, W > 65535 or
 * H > 65535; depth_tol not finite or < 0; min_cos outside [0, 1); z_near not finite or <= 0.  A vertex index outside
 * [0, n_vertices) is found on the device as in ps_mesh_render.  n_triangles = 0 is valid: nothing is written and the report
 * is zero.  Synchronous.
 * Workspace: 184 bytes per view. */
int ps_mesh_texture(int device, int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses,
                    const float* const* d_depth, const ps_mesh_vertex* d_vertices, int64_t n_vertices, const int32_t* d_triangles,
                    int64_t n_triangles, const ps_texture_params* prm, uint8_t* d_atlas, int32_t* d_view, ps_texture_report* report);

#ifdef __cplusplus
}
#endif

#endif
