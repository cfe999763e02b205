/* surfel_mesh.h -- C ABI of the GPU mesh extractor: TSDF fusion of rendered views and marching cubes (next-row:
 * LaRa's tools/meshExtractor.py, which runs open3d's ScalableTSDFVolume on the host).  Part of the same library and
 * ABI version as surfel_rasterizer.h; the same conventions hold (device pointers unless "host", int status, 0 = ok,
 * srf_last_error() on failure, only enqueues work on `stream`).
 *
 * The volume is a dense block of voxels n = n0 + (i, j, k), 0 <= i < dims[0] (x), j < dims[1] (y), k < dims[2] (z),
 * with linear index i + dims[0] (j + dims[1] k).  Voxel n's centre is (n + 0.5) voxel_size, so every block lies on one
 * grid aligned to the world origin.  Its state is SoA fp32: tsdf[N], weight[N], color[3][N] (0..255), N the voxel
 * count; the caller allocates it and clears it to 0 before the first integration.  A block of more than
 * 2^31 / SRF_MC_MAX_TRIS_BOUND voxels, or whose indices n reach 2^24 in magnitude, is rejected, so that every vertex,
 * triangle and voxel index the extractor forms fits in int32 and every voxel centre is exact in fp32.
 */
#ifndef SURFEL_MESH_H_
#define SURFEL_MESH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* one record per view: the world-to-camera matrix (row-major, OpenCV axes: x right, y down, z forward), the pinhole
 * intrinsics and the depth truncation, SRF_MESH_CAM_FLOATS floats each, the rest padding */
#define SRF_MESH_CAM_FLOATS 24
#define SRF_MESH_CAM_W2C 0
#define SRF_MESH_CAM_FX 16
#define SRF_MESH_CAM_FY 17
#define SRF_MESH_CAM_CX 18
#define SRF_MESH_CAM_CY 19
#define SRF_MESH_CAM_DEPTH_TRUNC 20
/* an upper bound of the triangles one cube can produce (the generated table's maximum is at most this) */
#define SRF_MC_MAX_TRIS_BOUND 5

/* Fuse V views into the block in place (open3d's legacy TSDF integration, DESIGN §3.15).  depth [V,H,W], acc [V,H,W]
 * and image [V,3,H,W] are the fused epilogue's planar outputs; cams [V][SRF_MESH_CAM_FLOATS].  A pixel whose acc is
 * < alpha_thres or whose depth is > the view's depth_trunc has no depth.  Each voxel applies the views in order, so two
 * calls with V1 and then V2 views give the same bits as one call with the V1 + V2 views.  n0, dims: host int[3]. */
int srf_tsdf_integrate(void* stream, const int* n0, const int* dims, float voxel_size, float sdf_trunc,
                       float* tsdf, float* weight, float* color,
                       int V, int H, int W, const float* depth, const float* acc, const float* image,
                       const float* cams, float alpha_thres);

/* Marching cubes over the block.  A cube is the 8 voxels n + {0,1}^3 (cube n is the one at its minimum corner), valid if
 * all 8 weights are > 0; a voxel is inside if its tsdf is < 0.  Each crossing edge of a valid cube carries one vertex,
 * shared by the cubes that use it; voxel n owns the three edges from n along +x, +y, +z.
 * srf_mesh_count classifies the cubes, marks the crossing edges and scans them: it writes the vertex count Nv and the
 * triangle count Nt to totals (device int32[2]) and keeps in the workspace (256-byte aligned,
 * srf_mesh_workspace_bytes) what srf_mesh_emit reads.  srf_mesh_emit then writes vertices [Nv,3], colors [Nv,3] (0..1)
 * and triangles [Nt,3] (int32 vertex indices) in a canonical order: vertices by (owning voxel, axis), triangles by
 * (cube, table order).  No float atomics: the output is bit-reproducible.  Pass both the same block and workspace,
 * and the totals srf_mesh_count wrote as Nv, Nt. */
int srf_mesh_workspace_bytes(const int* dims, size_t* bytes);
int srf_mesh_count(void* stream, const int* dims, const float* tsdf, const float* weight, void* workspace,
                   int32_t* totals);
int srf_mesh_emit(void* stream, const int* n0, const int* dims, float voxel_size, const float* tsdf,
                  const float* color, const void* workspace, int Nv, int Nt,
                  float* vertices, float* colors, int32_t* triangles);

/* LaRa's mesh postprocess (tools/meshExtractor.py:116-134) on the device, for vertices [Nv,3], colors [Nv,3] and
 * triangles [Nt,3] (int32).  With aabb (host double[6]: lo xyz, hi xyz; NULL = no crop) a triangle with a vertex outside
 * the inclusive box is dropped (each float coordinate compared as a double, a NaN is outside).  Two surviving triangles
 * are adjacent if they share an undirected vertex pair among their edges (a, b), (b, c), (c, a); the clusters are the
 * connected components.  With C clusters, every triangle whose cluster holds at least the min(C, keep)-th largest count
 * is kept (ties keep more), and a vertex is kept if a kept triangle references it.  Kept vertices, colours and triangles
 * stay in input order, the triangles' indices remapped.
 * srf_mesh_filter_count writes to totals (device int32[4]) the kept vertex count, the kept triangle count, the cluster
 * count after the crop and the number of triangles with an index outside [0, Nv), and keeps in the workspace (256-byte
 * aligned, srf_mesh_filter_workspace_bytes) what srf_mesh_filter_emit reads.  If the last count is not 0 the mesh is
 * invalid: such triangles are treated as cropped, and the caller should not emit.  srf_mesh_filter_emit then writes
 * out_vertices, out_colors [Nv_out,3] and out_triangles [Nt_out,3]; pass both the same inputs and workspace, and the
 * first two totals as Nv_out, Nt_out.  Integer atomics only: the output is bit-reproducible. */
int srf_mesh_filter_workspace_bytes(int Nv, int Nt, size_t* bytes);
int srf_mesh_filter_count(void* stream, int Nv, int Nt, const float* vertices, const int32_t* triangles,
                          const double* aabb, int keep, void* workspace, int32_t* totals);
int srf_mesh_filter_emit(void* stream, int Nv, int Nt, const float* vertices, const float* colors,
                         const int32_t* triangles, const void* workspace, int Nv_out, int Nt_out,
                         float* out_vertices, float* out_colors, int32_t* out_triangles);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_MESH_H_ */
