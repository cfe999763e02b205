// mesh.cu -- GPU mesh extraction for LaRa's tools/meshExtractor.py (DESIGN §3.15): TSDF fusion of V rendered views
// into a dense voxel block, then marching cubes with the generated table of mc_table.cuh.  The C entries of
// include/surfel_mesh.h are defined here.
//
// Integration, one thread per voxel applying the views in order (fp32, each step one rounding, in this order):
//   p     = (n + 0.5) * voxel_size                                   per axis
//   q_r   = ((E_r0 p0 + E_r1 p1) + E_r2 p2) + E_r3                  fmaf chain, r = 0..2 (camera x, y, z)
//   skip if !(q2 > 0)
//   u_f   = ((q0 * fx) / q2 + cx) + 0.5,  v_f likewise
//   skip unless 1e-4 <= u_f < W - 1e-4 and 1e-4 <= v_f < H - 1e-4;  u = (int)u_f, v = (int)v_f
//   skip if acc[v,u] < alpha_thres, depth[v,u] > depth_trunc or !(depth[v,u] > 0)
//   sdf   = (d - q2) * sqrt((1 + ((u - cx)/fx)^2) + ((v - cy)/fy)^2)
//   if sdf > -sdf_trunc: t = min(1, sdf / sdf_trunc); tsdf = (tsdf w + t) / (w + 1);
//                        c = (c w + trunc(255 rgb)) / (w + 1) per channel; w = w + 1
// The truncation of u_f to a pixel is the step that turns an ulp of the projection into a different depth sample.
//
// Marching cubes: count (classify + idempotent edge marks, then two exclusive scans over edges and cubes, totals to
// device memory) and emit (one thread per voxel writes the vertices of its three edges and the triangles of its
// cube).  Integer scans and stores only; every output lands at an index the scans fixed.
#include "../../include/surfel_mesh.h"
#include "mc_table.cuh"
#include "surfel_kernels.h"

static_assert(SRF_MC_MAX_TRIS <= SRF_MC_MAX_TRIS_BOUND, "the generated table exceeds the header's triangle bound");

namespace srf {
namespace {

constexpr int kMeshThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 4;
constexpr int kScanTile = kScanThreads * kScanItems;

struct Grid {
    int n0[3], d[3];
    size_t N;
};

__device__ __forceinline__ void voxel_ijk(const Grid& g, size_t idx, int& i, int& j, int& k) {
    i = (int)(idx % (size_t)g.d[0]);
    const size_t r = idx / (size_t)g.d[0];
    j = (int)(r % (size_t)g.d[1]);
    k = (int)(r / (size_t)g.d[1]);
}

__device__ __forceinline__ float centre(int n, float vs) { return __fmul_rn(__fadd_rn((float)n, 0.5f), vs); }

struct IntegrateArgs {
    Grid g;
    float vs, sdf_trunc, alpha_thres;
    int V, H, W;
    float* tsdf; float* weight; float* color;
    const float* depth; const float* acc; const float* image; const float* cams;
};

__global__ void __launch_bounds__(kMeshThreads) tsdf_integrate_kernel(IntegrateArgs a) {
    const size_t idx = (size_t)blockIdx.x * kMeshThreads + threadIdx.x;
    if (idx >= a.g.N) return;
    int i, j, k;
    voxel_ijk(a.g, idx, i, j, k);
    const float p0 = centre(a.g.n0[0] + i, a.vs), p1 = centre(a.g.n0[1] + j, a.vs), p2 = centre(a.g.n0[2] + k, a.vs);
    const size_t HW = (size_t)a.H * a.W, N = a.g.N;
    const float umax = __fsub_rn((float)a.W, 0.0001f), vmax = __fsub_rn((float)a.H, 0.0001f);
    float tsdf = a.tsdf[idx], w = a.weight[idx];
    float c0 = a.color[idx], c1 = a.color[N + idx], c2 = a.color[2 * N + idx];
    bool changed = false;
    for (int v = 0; v < a.V; ++v) {
        const float* cam = a.cams + (size_t)v * SRF_MESH_CAM_FLOATS;
        float q[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float* E = cam + SRF_MESH_CAM_W2C + 4 * r;
            q[r] = __fadd_rn(__fmaf_rn(__ldg(E + 2), p2, __fmaf_rn(__ldg(E + 1), p1, __fmul_rn(__ldg(E), p0))), __ldg(E + 3));
        }
        if (!(q[2] > 0.0f)) continue;
        const float fx = __ldg(cam + SRF_MESH_CAM_FX), fy = __ldg(cam + SRF_MESH_CAM_FY);
        const float cx = __ldg(cam + SRF_MESH_CAM_CX), cy = __ldg(cam + SRF_MESH_CAM_CY);
        const float uf = __fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(q[0], fx), q[2]), cx), 0.5f);
        const float vf = __fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(q[1], fy), q[2]), cy), 0.5f);
        if (!(uf >= 0.0001f && uf < umax && vf >= 0.0001f && vf < vmax)) continue;
        const int u = (int)uf, vv = (int)vf;
        const size_t pix = (size_t)v * HW + (size_t)vv * a.W + u;
        if (__ldg(a.acc + pix) < a.alpha_thres) continue;
        const float d = __ldg(a.depth + pix);
        if (d > __ldg(cam + SRF_MESH_CAM_DEPTH_TRUNC) || !(d > 0.0f)) continue;
        const float ru = __fdiv_rn(__fsub_rn((float)u, cx), fx), rv = __fdiv_rn(__fsub_rn((float)vv, cy), fy);
        const float mult = __fsqrt_rn(__fadd_rn(__fadd_rn(1.0f, __fmul_rn(ru, ru)), __fmul_rn(rv, rv)));
        const float sdf = __fmul_rn(__fsub_rn(d, q[2]), mult);
        if (!(sdf > -a.sdf_trunc)) continue;
        const float t = fminf(1.0f, __fdiv_rn(sdf, a.sdf_trunc));
        const float w1 = __fadd_rn(w, 1.0f);
        tsdf = __fdiv_rn(__fadd_rn(__fmul_rn(tsdf, w), t), w1);
        const float* img = a.image + (size_t)v * 3 * HW + (size_t)vv * a.W + u;
        c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, w), truncf(__fmul_rn(__ldg(img), 255.0f))), w1);
        c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, w), truncf(__fmul_rn(__ldg(img + HW), 255.0f))), w1);
        c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, w), truncf(__fmul_rn(__ldg(img + 2 * HW), 255.0f))), w1);
        w = w1;
        changed = true;
    }
    if (changed) {
        a.tsdf[idx] = tsdf;
        a.weight[idx] = w;
        a.color[idx] = c0; a.color[N + idx] = c1; a.color[2 * N + idx] = c2;
    }
}

// ---- marching cubes ----

struct Workspace { size_t edge, tri, cases, sums, total; size_t n_edge, n_cube, nb_edge, nb_cube; };

Workspace workspace_layout(size_t N) {
    Workspace l;
    l.n_edge = 3 * N;
    l.n_cube = N;
    l.nb_edge = (l.n_edge + kScanTile - 1) / kScanTile;
    l.nb_cube = (l.n_cube + kScanTile - 1) / kScanTile;
    l.edge = 0;                                             // u32 [3N + 1]: crossing flags, then vertex ids; [3N] = Nv
    l.tri = align_up(l.edge + 4 * (l.n_edge + 1));          // u32 [N + 1]: triangle counts, then offsets;  [N] = Nt
    l.cases = align_up(l.tri + 4 * (l.n_cube + 1));         // u8 [N]: sign case of each valid cube, 0 otherwise
    l.sums = align_up(l.cases + l.n_cube);                  // u32 [nb_edge + nb_cube]: per-tile sums of the scans
    l.total = align_up(l.sums + 4 * (l.nb_edge + l.nb_cube));
    return l;
}

// corner c's voxel offset along each axis, and local edge e's start corner and axis (tools/gen_mc_table.py)
__device__ __forceinline__ void edge_start(int e, int& c, int& axis) {
    axis = e >> 2;
    const int b = e & 3;
    const int o0 = axis == 0 ? 1 : 0, o1 = axis == 2 ? 1 : 2;
    c = ((b & 1) << o0) | (((b >> 1) & 1) << o1);
}

__device__ __forceinline__ size_t corner_index(const Grid& g, size_t idx, int c) {
    return idx + (size_t)(c & 1) + ((c >> 1) & 1) * (size_t)g.d[0] + ((c >> 2) & 1) * (size_t)g.d[0] * g.d[1];
}

struct CountArgs {
    Grid g;
    const float* tsdf; const float* weight;
    uint32_t* edge; uint32_t* tri; uint8_t* cases;
};

__global__ void __launch_bounds__(kMeshThreads) mesh_classify_kernel(CountArgs a) {
    const size_t idx = (size_t)blockIdx.x * kMeshThreads + threadIdx.x;
    if (idx >= a.g.N) return;
    int i, j, k;
    voxel_ijk(a.g, idx, i, j, k);
    uint32_t ntri = 0;
    int cs = 0;
    if (i + 1 < a.g.d[0] && j + 1 < a.g.d[1] && k + 1 < a.g.d[2]) {
        bool valid = true;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const size_t ci = corner_index(a.g, idx, c);
            valid &= __ldg(a.weight + ci) > 0.0f;
            cs |= (__ldg(a.tsdf + ci) < 0.0f ? 1 : 0) << c;
        }
        if (!valid) cs = 0;
        ntri = kMcTriCount[cs];
        if (ntri) {
#pragma unroll
            for (int e = 0; e < 12; ++e) {
                int c, axis;
                edge_start(e, c, axis);
                if (((cs >> c) & 1) != ((cs >> (c | (1 << axis))) & 1))
                    a.edge[3 * corner_index(a.g, idx, c) + axis] = 1u;     // idempotent: any cube sharing it stores 1
            }
        }
    }
    a.tri[idx] = ntri;
    a.cases[idx] = (uint8_t)cs;
}

// exclusive scan of u32 data[0, n) in tiles of kScanTile, in place; data[n] receives the total
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t x, uint32_t* warp_sums, uint32_t& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t s = lane < kScanThreads / 32 ? warp_sums[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        warp_sums[lane] = s;                               // inclusive over warps
    }
    __syncthreads();
    total = warp_sums[kScanThreads / 32 - 1];
    const uint32_t before = wid ? warp_sums[wid - 1] : 0u;
    __syncthreads();                                       // warp_sums is reused by the next call
    return before + inc - x;
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_sums_kernel(const uint32_t* data, size_t n, uint32_t* sums) {
    __shared__ uint32_t ws[32];
    const size_t base = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanItems;
    uint32_t s = 0;
#pragma unroll
    for (int q = 0; q < kScanItems; ++q) s += base + q < n ? data[base + q] : 0u;
    uint32_t total;
    block_exclusive_scan(s, ws, total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) scan_sums_kernel(uint32_t* sums, size_t nb, uint32_t* data_end,
                                                                 int32_t* total_out) {
    __shared__ uint32_t ws[32];
    uint32_t carry = 0;
    for (size_t b0 = 0; b0 < nb; b0 += kScanThreads) {
        const size_t b = b0 + threadIdx.x;
        const uint32_t x = b < nb ? sums[b] : 0u;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan(x, ws, total);
        if (b < nb) sums[b] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        *data_end = carry;
        *total_out = (int32_t)carry;
    }
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(uint32_t* data, size_t n, const uint32_t* sums) {
    __shared__ uint32_t ws[32];
    const size_t base = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanItems;
    uint32_t v[kScanItems], s = 0;
#pragma unroll
    for (int q = 0; q < kScanItems; ++q) {
        v[q] = base + q < n ? data[base + q] : 0u;
        s += v[q];
    }
    uint32_t total;
    uint32_t run = block_exclusive_scan(s, ws, total) + sums[blockIdx.x];
#pragma unroll
    for (int q = 0; q < kScanItems; ++q) {
        if (base + q < n) data[base + q] = run;
        run += v[q];
    }
}

cudaError_t exclusive_scan(uint32_t* data, size_t n, uint32_t* sums, size_t nb, int32_t* total, cudaStream_t stream) {
    scan_tile_sums_kernel<<<(unsigned)nb, kScanThreads, 0, stream>>>(data, n, sums);
    scan_sums_kernel<<<1, kScanThreads, 0, stream>>>(sums, nb, data + n, total);
    scan_apply_kernel<<<(unsigned)nb, kScanThreads, 0, stream>>>(data, n, sums);
    return cudaGetLastError();
}

struct EmitArgs {
    Grid g;
    float vs;
    const float* tsdf; const float* color;
    const uint32_t* edge; const uint32_t* tri; const uint8_t* cases;
    float* vertices; float* colors; int32_t* triangles;
};

__global__ void __launch_bounds__(kMeshThreads) mesh_emit_kernel(EmitArgs a) {
    const size_t idx = (size_t)blockIdx.x * kMeshThreads + threadIdx.x;
    if (idx >= a.g.N) return;
    int ijk[3];
    voxel_ijk(a.g, idx, ijk[0], ijk[1], ijk[2]);
    const size_t N = a.g.N;
#pragma unroll
    for (int axis = 0; axis < 3; ++axis) {
        const size_t e = 3 * idx + axis;
        const uint32_t id = a.edge[e];
        if (a.edge[e + 1] == id) continue;                 // not a crossing edge of a valid cube
        const size_t other = corner_index(a.g, idx, 1 << axis);
        const float t0 = __ldg(a.tsdf + idx), t1 = __ldg(a.tsdf + other);
        const float f0 = fabsf(t0), f1 = fabsf(t1), s = __fadd_rn(f0, f1);
        float* vx = a.vertices + 3 * (size_t)id;
        float* cl = a.colors + 3 * (size_t)id;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            float p = centre(a.g.n0[r] + ijk[r], a.vs);
            if (r == axis) p = __fadd_rn(p, __fmul_rn(__fdiv_rn(f0, s), a.vs));
            vx[r] = p;
            const float cs = __ldg(a.color + r * N + idx), ce = __ldg(a.color + r * N + other);
            cl[r] = __fdiv_rn(__fdiv_rn(__fadd_rn(__fmul_rn(f1, cs), __fmul_rn(f0, ce)), s), 255.0f);
        }
    }
    const uint32_t t0 = a.tri[idx], nt = a.tri[idx + 1] - t0;
    if (!nt) return;
    const int cs = a.cases[idx];
    int32_t* out = a.triangles + 3 * (size_t)t0;
    for (uint32_t t = 0; t < 3 * nt; ++t) {
        int c, axis;
        edge_start(kMcTris[cs][t], c, axis);
        out[t] = (int32_t)a.edge[3 * corner_index(a.g, idx, c) + axis];
    }
}

int check_grid(const char* fn, const int* n0, const int* dims, Grid& g) {
    if (!dims) return set_error("%s: null dims", fn);
    for (int r = 0; r < 3; ++r) {
        if (dims[r] <= 0) return set_error("%s: bad dims (%d, %d, %d)", fn, dims[0], dims[1], dims[2]);
        g.d[r] = dims[r];
        g.n0[r] = n0 ? n0[r] : 0;
        if ((long long)g.n0[r] <= -(1ll << 24) || (long long)g.n0[r] + dims[r] >= (1ll << 24))
            return set_error("%s: voxel indices must stay within +-2^24 (n0 = %d, dims = %d on axis %d)", fn, g.n0[r],
                             dims[r], r);
    }
    g.N = (size_t)dims[0] * dims[1] * dims[2];
    if (g.N > (size_t)INT32_MAX / SRF_MC_MAX_TRIS_BOUND)
        return set_error("%s: a block of %zu voxels is over the limit of %d (vertex and triangle indices are int32)", fn,
                         g.N, INT32_MAX / SRF_MC_MAX_TRIS_BOUND);
    return 0;
}

}  // namespace
}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_tsdf_integrate(void* stream, const int* n0, const int* dims, float voxel_size, float sdf_trunc,
                                  float* tsdf, float* weight, float* color, int V, int H, int W, const float* depth,
                                  const float* acc, const float* image, const float* cams, float alpha_thres) {
    const char* fn = "srf_tsdf_integrate";
    srf::IntegrateArgs a;
    if (!n0) return set_error("%s: null n0", fn);
    if (srf::check_grid(fn, n0, dims, a.g)) return 1;
    if (V < 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (V=%d, H=%d, W=%d)", fn, V, H, W);
    if (H > (1 << 24) || W > (1 << 24)) return set_error("%s: image too large", fn);
    if (!(voxel_size > 0.0f) || !(voxel_size < 1e30f) || !(sdf_trunc > 0.0f) || !(sdf_trunc < 1e30f))
        return set_error("%s: voxel_size and sdf_trunc must be positive and finite", fn);
    if (!tsdf || !weight || !color) return set_error("%s: null volume pointer", fn);
    if (V > 0 && (!depth || !acc || !image || !cams)) return set_error("%s: null view pointer", fn);
    if (V == 0) return 0;
    a.vs = voxel_size; a.sdf_trunc = sdf_trunc; a.alpha_thres = alpha_thres;
    a.V = V; a.H = H; a.W = W;
    a.tsdf = tsdf; a.weight = weight; a.color = color;
    a.depth = depth; a.acc = acc; a.image = image; a.cams = cams;
    const size_t blocks = (a.g.N + srf::kMeshThreads - 1) / srf::kMeshThreads;
    srf::tsdf_integrate_kernel<<<(unsigned)blocks, srf::kMeshThreads, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("tsdf_integrate launch", e);
}

extern "C" int srf_mesh_workspace_bytes(const int* dims, size_t* bytes) {
    srf::Grid g;
    if (srf::check_grid("srf_mesh_workspace_bytes", nullptr, dims, g)) return 1;
    if (!bytes) return set_error("srf_mesh_workspace_bytes: null output");
    *bytes = srf::workspace_layout(g.N).total;
    return 0;
}

extern "C" int srf_mesh_count(void* stream_, const int* dims, const float* tsdf, const float* weight, void* workspace,
                              int32_t* totals) {
    const char* fn = "srf_mesh_count";
    srf::CountArgs a;
    if (srf::check_grid(fn, nullptr, dims, a.g)) return 1;
    if (!tsdf || !weight || !totals) return set_error("%s: null pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const cudaStream_t stream = (cudaStream_t)stream_;
    const srf::Workspace l = srf::workspace_layout(a.g.N);
    char* ws = static_cast<char*>(workspace);
    a.tsdf = tsdf; a.weight = weight;
    a.edge = reinterpret_cast<uint32_t*>(ws + l.edge);
    a.tri = reinterpret_cast<uint32_t*>(ws + l.tri);
    a.cases = reinterpret_cast<uint8_t*>(ws + l.cases);
    uint32_t* sums = reinterpret_cast<uint32_t*>(ws + l.sums);
    cudaError_t e = cudaMemsetAsync(a.edge, 0, 4 * l.n_edge, stream);
    if (e != cudaSuccess) return cuda_error("memset mesh edge flags", e);
    const size_t blocks = (a.g.N + srf::kMeshThreads - 1) / srf::kMeshThreads;
    srf::mesh_classify_kernel<<<(unsigned)blocks, srf::kMeshThreads, 0, stream>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error("mesh_classify launch", e);
    if ((e = srf::exclusive_scan(a.edge, l.n_edge, sums, l.nb_edge, totals, stream)) != cudaSuccess ||
        (e = srf::exclusive_scan(a.tri, l.n_cube, sums + l.nb_edge, l.nb_cube, totals + 1, stream)) != cudaSuccess)
        return cuda_error("mesh scan launch", e);
    return 0;
}

extern "C" int srf_mesh_emit(void* stream, const int* n0, const int* dims, float voxel_size, const float* tsdf,
                             const float* color, const void* workspace, int Nv, int Nt,
                             float* vertices, float* colors, int32_t* triangles) {
    const char* fn = "srf_mesh_emit";
    srf::EmitArgs a;
    if (!n0) return set_error("%s: null n0", fn);
    if (srf::check_grid(fn, n0, dims, a.g)) return 1;
    if (!(voxel_size > 0.0f) || !(voxel_size < 1e30f)) return set_error("%s: voxel_size must be positive and finite", fn);
    if (!tsdf || !color) return set_error("%s: null volume pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    if (Nv < 0 || Nt < 0) return set_error("%s: bad totals (Nv=%d, Nt=%d)", fn, Nv, Nt);
    if ((Nv > 0 && (!vertices || !colors)) || (Nt > 0 && !triangles)) return set_error("%s: null output pointer", fn);
    if (Nv == 0 && Nt == 0) return 0;
    const srf::Workspace l = srf::workspace_layout(a.g.N);
    const char* ws = static_cast<const char*>(workspace);
    a.vs = voxel_size;
    a.tsdf = tsdf; a.color = color;
    a.edge = reinterpret_cast<const uint32_t*>(ws + l.edge);
    a.tri = reinterpret_cast<const uint32_t*>(ws + l.tri);
    a.cases = reinterpret_cast<const uint8_t*>(ws + l.cases);
    a.vertices = vertices; a.colors = colors; a.triangles = triangles;
    const size_t blocks = (a.g.N + srf::kMeshThreads - 1) / srf::kMeshThreads;
    srf::mesh_emit_kernel<<<(unsigned)blocks, srf::kMeshThreads, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("mesh_emit launch", e);
}
