/* Surface meshes (an addition to the reference's interface): depth maps fused into a dense truncated signed distance
 * volume, and a watertight triangle mesh extracted from it by marching tetrahedra.
 *
 * ps_depth_maps / ps_depth_filter end with one depth map per reference and a point cloud in which a surface point appears
 * once per reference that sees it.  The next step of every photogrammetry pipeline is a surface: AliceVision's Meshing
 * node follows DepthMapFilter, COLMAP follows stereo_fusion with its Poisson and Delaunay meshers.  Volumetric fusion
 * (Curless and Levoy 1996) keeps every step data-parallel and deterministic: each voxel folds the views in a fixed order
 * with no floating-point atomics, and extraction is a classification, integer scans, a radix sort and a compaction.
 *
 * Declared apart from popsift_b200.h; same library, same ABI version. */
#ifndef POPSIFT_B200_MESH_H
#define POPSIFT_B200_MESH_H

#include "popsift_b200_depth.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ps_volume {                /* 72 bytes, HOST struct describing DEVICE voxels                            */
    double origin[3];                     /* world position of grid point (0, 0, 0), finite                            */
    double voxel;                         /* grid spacing, finite and > 0                                              */
    int32_t nx, ny, nz, pad_;             /* grid points per axis, 2 .. 2048 each, nx ny nz < 2^31; pad_ ignored       */
    float* tsdf;                          /* DEVICE, nx ny nz each, grid point (i, j, k) at index i + nx (j + ny k)    */
    float* weight;
    float* grey;
} ps_volume;

typedef struct ps_tsdf_params {           /* 8 bytes */
    float   trunc;                        /* truncation distance, world units, finite and > 0                          */
    int32_t min_consistent;               /* 0 .. 255; > 0: a pixel needs n_consistent >= min_consistent               */
} ps_tsdf_params;

typedef struct ps_mesh_params {           /* 8 bytes */
    float   min_weight;                   /* a cell is meshed when its 8 corners have weight >= min_weight, finite > 0 */
    int32_t pad_;                         /* ignored                                                                   */
} ps_mesh_params;

typedef struct ps_mesh_vertex {           /* 16 bytes, DEVICE */
    float X[3];                           /* world position                                                            */
    float grey;                           /* interpolated grey level                                                   */
} ps_mesh_vertex;

typedef struct ps_tsdf_report {           /* 16 bytes, HOST */
    int64_t n_updates;                    /* (grid point, view) updates of step 6                                      */
    int64_t n_voxels_touched;             /* grid points with at least one update                                      */
} ps_tsdf_report;

typedef struct ps_mesh_report {           /* 24 bytes, HOST */
    int64_t n_cells;                      /* meshed cells with a sign change                                           */
    int64_t n_vertices;
    int64_t n_triangles;
} ps_mesh_report;

/* Sets tsdf, weight and grey of every grid point to 0.  A new volume is cleared before its first integration; the library
 * never reads a volume from the host.  Errors: PS_ERR_ARG for a volume ps_tsdf_integrate refuses.  Synchronous. */
int ps_volume_clear(int device, const ps_volume* vol);

/* Folds depth maps into the volume.  View v (0 .. n_views - 1) is the grey image images[v] (HOST array of structs whose
 * data is DEVICE memory), camera cams[v], world-to-camera pose poses[v] (X_cam = R X + t) and d_depth[v] (HOST array of
 * DEVICE pointers): a float map of images[v]'s width x height, row stride width, as ps_depth_maps writes it; d_depth <= 0
 * marks an unknown pixel.  d_n_consistent[v] (uint8, same layout, ps_depth_filter's output) is read only when
 * min_consistent > 0; the array may be NULL when min_consistent == 0.  For every grid point g = (i, j, k),
 * X_g = origin + voxel (i, j, k) in double, and for v = 0 .. n_views - 1 in this order:
 *   1. X_c = R_v X_g + t_v in double, each row as ((R_r0 X + R_r1 Y) + R_r2 Z) + t_r.  The view is skipped unless
 *      X_c.z > 0.
 *   2. pi = (fx X_c.x / X_c.z + cx, fy X_c.y / X_c.z + cy) as in ps_depth_filter, in double; q = floor(pi + 1/2) per
 *      coordinate must lie inside the image: 0 <= q_x < w, 0 <= q_y < h.
 *   3. D = d_depth_v(q) must be > 0; when min_consistent > 0, n_consistent_v(q) >= min_consistent too.
 *   4. sdf = D - X_c.z in double; the view is skipped when sdf < -trunc.
 *   5. tau = (float) min(1, sdf / trunc), the division in double.
 *   6. In float, in this order: W' = W + 1; T' = (T W + tau) / W'; G' = (G W + I_v(q)) / W'.
 * An unknown pixel changes nothing.  Free space in front of a surface gets tau = 1 from every view that sees through it,
 * which is what removes floaters; grid points more than trunc behind the observed surface keep their values.
 * The fold is sequential per grid point and views never interact, so integrating views A and then views B gives the same
 * bytes as one call with A followed by B, and two identical calls give identical bytes (no floating-point atomics).
 * *report: the (grid point, view) updates of step 6 and the grid points with at least one.
 * Errors: PS_ERR_ARG before any device work, with the volume and *report untouched, for: n_views < 0; NULL prm, vol or
 * report, or (n_views > 0) NULL images, cams, poses or d_depth, or d_n_consistent NULL with min_consistent > 0; a volume
 * whose origin or voxel is not finite, voxel <= 0, a dimension outside 2 .. 2048, nx ny nz >= 2^31, or an array that is
 * not device memory on `device` or overlaps another; trunc not finite or <= 0; min_consistent outside 0 .. 255; a camera
 * or pose ps_triangulate_tracks refuses; an image ps_depth_filter refuses (data not device memory on `device`, width or
 * height outside 1 .. 65535, pitch < width); a d_depth or used d_n_consistent entry that is not device memory on
 * `device`.  n_views = 0 is valid: the volume is untouched and the report zero.  Synchronous.
 * Workspace: 168 bytes per view. */
int ps_tsdf_integrate(int device, int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses,
                      const float* const* d_depth, const uint8_t* const* d_n_consistent, const ps_tsdf_params* prm,
                      const ps_volume* vol, ps_tsdf_report* report);

/* Extracts the surface T = 0 by marching tetrahedra over the Kuhn (Freudenthal) split of every cell.  A cell is the cube
 * of grid points (i, j, k) + e, e in {0, 1}^3, i < nx - 1, j < ny - 1, k < nz - 1, with corner code c = e_x + 2 e_y + 4 e_z;
 * its index is that of its corner 0.  A corner is inside when T < 0 and outside when T >= 0 (NaN is outside).
 *   1. Cells: a cell is meshed when all 8 corners have weight >= min_weight, and active when it is meshed and has both
 *      inside and outside corners.
 *   2. Split: for each permutation (a, b, c) of the axes in lexicographic order, the tetrahedron of the corners
 *      0, e_a, e_a + e_b, (1, 1, 1); for odd permutations the second and third corners are swapped, so every tetrahedron
 *      is positively oriented.  Every face of a cell is split along the diagonal from its lowest to its highest corner,
 *      the same in both cells that share it, so the mesh is watertight by construction.
 *   3. Edges: every edge of a tetrahedron joins a lower corner a to an upper corner b = a + d with d one of the 7 nonzero
 *      0/1 vectors (3 axes, 3 face diagonals, the body diagonal); its code is d_x + 2 d_y + 4 d_z, and its key
 *      8 (index of a) + code.  A cell has 19 distinct edges.
 *   4. Triangles, per tetrahedron with local corners 0 .. 3 in the order of step 2: 1 inside corner a gives the triangle
 *      on its three edges to the outside corners, in local order; 3 inside corners give the triangle on the edges from
 *      them to the outside corner b, in local order; 2 inside corners a < b with outside corners c < d give the quad
 *      (ac, ad, bd, bc) split along the diagonal ac-bd into (ac, ad, bd) and (ac, bd, bc).  Each triangle is then
 *      ordered so that its normal (v1 - v0) x (v2 - v0) points from the inside corners to the outside corners: towards
 *      the cameras.  The table this rule gives is kTetTri in k_mesh.h.  Marching tetrahedra needs no case table with
 *      ambiguous faces, at the cost of about twice the triangles of marching cubes.
 *   5. Vertices: exactly the edges some triangle references, ordered by key.  With o = (float) origin and h = (float)
 *      voxel, an edge's vertex is computed from its lower endpoint, in float, in this order: s = T_a / (T_a - T_b);
 *      X_c = o_c + h ((float) a_c + s d_c) per axis; grey = G_a + s (G_b - G_a).
 *   6. Outputs: d_vertices[0 .. n_vertices - 1] and d_triangles[3 m .. 3 m + 2] (int32 vertex indices) for the triangles
 *      in (cell index, tetrahedron, triangle) order.  *report: the active cells, the vertices and the triangles.
 * When n_vertices > max_vertices, n_triangles > max_triangles or n_vertices >= 2^31, the call returns PS_ERR_OVERFLOW
 * with *report set and the outputs untouched (n_vertices = -1 when the cells list 2^31 or more edge entries); a
 * count-only call passes NULL outputs with capacity 0.  Deterministic: integer scans, a stable radix sort, no atomics on
 * floats; two identical calls give identical bytes.
 * Errors: PS_ERR_ARG before any device work, with the outputs and *report untouched, for: NULL vol, prm or report; a volume
 * ps_tsdf_integrate refuses; min_weight not finite or <= 0; a capacity < 0; an output that is not device memory on
 * `device` with its capacity > 0.  Synchronous; two small read-backs: the classification's totals, which size the
 * workspace, and the vertex count.
 * Workspace: O(surface): 12 bytes per active cell and about 24 per edge entry (at most 19 per active cell), plus 24 bytes
 * per 2048 grid points for the block counts. */
int ps_tsdf_mesh(int device, const ps_volume* vol, const ps_mesh_params* prm, int64_t max_vertices, int64_t max_triangles,
                 ps_mesh_vertex* d_vertices, int32_t* d_triangles, ps_mesh_report* report);

#ifdef __cplusplus
}
#endif

#endif
