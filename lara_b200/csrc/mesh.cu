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
//
// Cluster filter (LaRa's postprocess): crop flags, an open-addressing hash table of the live triangles' undirected edges
// whose slots keep the smallest triangle on the edge, a union-find over "shares an edge" (larger root hooked under the
// smaller), component sizes, an exact radix select of the min(C, keep)-th largest size, then keep / used flags, the two
// scans and emit.  Integer atomics only, and every step's result is independent of scheduling: each component's
// root is its smallest triangle.
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

// n = 0 (nb = 0) only writes the total 0
cudaError_t exclusive_scan(uint32_t* data, size_t n, uint32_t* sums, size_t nb, int32_t* total, cudaStream_t stream) {
    if (nb) scan_tile_sums_kernel<<<(unsigned)nb, kScanThreads, 0, stream>>>(data, n, sums);
    scan_sums_kernel<<<1, kScanThreads, 0, stream>>>(sums, nb, data + n, total);
    if (nb) scan_apply_kernel<<<(unsigned)nb, kScanThreads, 0, stream>>>(data, n, sums);
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

// ---- cluster filter ----

constexpr unsigned long long kEmptyKey = ~0ull;    // no edge key: indices are < 2^31
constexpr uint32_t kDead = ~0u;                    // label of a cropped (or invalid) triangle
constexpr int kSelectPasses = 4;                   // 8-bit digits of a u32 cluster size

struct FilterWorkspace {
    size_t keys, owner, parent, size, label, used, hist, sel, sums, total;
    size_t slots, nb_tri, nb_vert;
};

FilterWorkspace filter_layout(size_t Nv, size_t Nt) {
    FilterWorkspace l;
    l.slots = 1;
    while (l.slots < 6 * Nt) l.slots <<= 1;                // load factor <= 1/2 over the 3 Nt edges
    l.nb_tri = (Nt + kScanTile - 1) / kScanTile;
    l.nb_vert = (Nv + kScanTile - 1) / kScanTile;
    l.keys = 0;                                             // u64 [slots]: edge keys min << 32 | max, ~0 = empty
    l.owner = align_up(l.keys + 8 * l.slots);               // u32 [slots]: smallest live triangle on the edge
    l.parent = align_up(l.owner + 4 * l.slots);             // i32 [Nt]: union-find forest, -1 = dropped by the crop
    l.size = align_up(l.parent + 4 * Nt);                   // u32 [Nt]: triangle count of each root
    l.label = align_up(l.size + 4 * Nt);                    // u32 [Nt + 1]: root, then keep flags, then offsets
    l.used = align_up(l.label + 4 * (Nt + 1));              // u32 [Nv + 1]: used flags, then offsets
    l.hist = align_up(l.used + 4 * (Nv + 1));               // u32 [4][256]: radix-select histograms
    l.sel = align_up(l.hist + 4 * 256 * kSelectPasses);     // u32 [2]: size prefix found so far, rank left in it
    l.sums = align_up(l.sel + 8);                           // u32 [nb_tri + nb_vert]: per-tile sums of the scans
    l.total = align_up(l.sums + 4 * (l.nb_tri + l.nb_vert));
    return l;
}

struct FilterArgs {
    int Nv, Nt, keep, crop;
    double lo[3], hi[3];
    size_t mask;                                            // slots - 1
    const float* vertices; const int32_t* triangles;
    unsigned long long* keys; uint32_t* owner; int32_t* parent; uint32_t* size; uint32_t* label; uint32_t* used;
    uint32_t* hist; uint32_t* sel; int32_t* totals;
};

__device__ __forceinline__ unsigned long long edge_key(int32_t x, int32_t y) {
    return x < y ? ((unsigned long long)x << 32) | (uint32_t)y : ((unsigned long long)y << 32) | (uint32_t)x;
}

__device__ __forceinline__ size_t edge_slot(unsigned long long k, size_t mask) {   // murmur3's 64-bit finaliser
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (size_t)k & mask;
}

__device__ __forceinline__ bool in_box(const FilterArgs& a, int32_t v) {
    const float* p = a.vertices + 3 * (size_t)v;
    bool in = true;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double x = (double)__ldg(p + r);
        in &= x >= a.lo[r] && x <= a.hi[r];                 // false for NaN
    }
    return in;
}

__global__ void __launch_bounds__(kMeshThreads) filter_crop_kernel(FilterArgs a) {
    const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (t >= a.Nt) return;
    const int32_t* tri = a.triangles + 3 * (size_t)t;
    const int32_t x = __ldg(tri), y = __ldg(tri + 1), z = __ldg(tri + 2);
    bool live;
    if ((uint32_t)x >= (uint32_t)a.Nv || (uint32_t)y >= (uint32_t)a.Nv || (uint32_t)z >= (uint32_t)a.Nv) {
        atomicAdd(a.totals + 3, 1);
        live = false;
    } else {
        live = !a.crop || (in_box(a, x) && in_box(a, y) && in_box(a, z));
    }
    a.parent[t] = live ? (int32_t)t : -1;
}

// pass one: every live triangle's three edges into the table; a slot's owner ends as the smallest triangle on its edge
__global__ void __launch_bounds__(kMeshThreads) filter_insert_kernel(FilterArgs a) {
    const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (t >= a.Nt || a.parent[t] < 0) return;
    const int32_t* tri = a.triangles + 3 * (size_t)t;
    const int32_t v[3] = {__ldg(tri), __ldg(tri + 1), __ldg(tri + 2)};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const unsigned long long key = edge_key(v[e], v[e == 2 ? 0 : e + 1]);
        for (size_t h = edge_slot(key, a.mask);; h = (h + 1) & a.mask) {
            const unsigned long long prev = atomicCAS(a.keys + h, kEmptyKey, key);
            if (prev == kEmptyKey || prev == key) {
                atomicMin(a.owner + h, (uint32_t)t);
                break;
            }
        }
    }
}

// root of x with path splitting (ECL-CC): every parent is <= its child, so a root is its component's smallest triangle
__device__ __forceinline__ int32_t find_root(volatile int32_t* parent, int32_t x) {
    int32_t cur = parent[x];
    if (cur != x) {
        int32_t next, prev = x;
        while (cur > (next = parent[cur])) {
            parent[prev] = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

// pass two: each live triangle joins the owners of its edges, hooking the larger root under the smaller
__global__ void __launch_bounds__(kMeshThreads) filter_union_kernel(FilterArgs a) {
    const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (t >= a.Nt || a.parent[t] < 0) return;
    const int32_t* tri = a.triangles + 3 * (size_t)t;
    const int32_t v[3] = {__ldg(tri), __ldg(tri + 1), __ldg(tri + 2)};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const unsigned long long key = edge_key(v[e], v[e == 2 ? 0 : e + 1]);
        size_t h = edge_slot(key, a.mask);
        while (a.keys[h] != key) h = (h + 1) & a.mask;
        const int32_t o = (int32_t)a.owner[h];
        if (o == t) continue;
        int32_t ra = find_root(a.parent, (int32_t)t), rb = find_root(a.parent, o);
        while (ra != rb) {
            if (ra > rb) { const int32_t s = ra; ra = rb; rb = s; }
            const int32_t prev = atomicCAS(a.parent + rb, rb, ra);
            if (prev == rb) break;
            rb = prev;                                      // rb was hooked meanwhile: retry from its new parent
        }
    }
}

// every live triangle's root into label, the roots' sizes and the cluster count
__global__ void __launch_bounds__(kMeshThreads) filter_label_kernel(FilterArgs a) {
    const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (t >= a.Nt) return;
    if (a.parent[t] < 0) {
        a.label[t] = kDead;
        return;
    }
    const int32_t r = find_root(a.parent, (int32_t)t);
    a.label[t] = (uint32_t)r;
    const unsigned peers = __match_any_sync(__activemask(), r);     // neighbours are mostly in one cluster
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(a.size + r, (uint32_t)__popc(peers));
    if (r == t) atomicAdd(a.totals + 2, 1);
}

// one thread: pass < 0 sets the rank min(C, keep); pass p fixes digit p (most significant first) of that rank's size
__global__ void filter_select_kernel(FilterArgs a, int pass) {
    if (pass < 0) {
        a.sel[0] = 0;
        a.sel[1] = min((uint32_t)a.totals[2], (uint32_t)a.keep);
        return;
    }
    const uint32_t k = a.sel[1];
    if (!k) return;
    const uint32_t* h = a.hist + 256 * pass;
    uint32_t cum = 0;
    for (int d = 255; d >= 0; --d) {
        if (cum + h[d] >= k) {
            a.sel[0] |= (uint32_t)d << (24 - 8 * pass);
            a.sel[1] = k - cum;
            return;
        }
        cum += h[d];
    }
}

// histogram of digit `pass` over the roots whose higher digits equal the prefix found so far
__global__ void __launch_bounds__(kMeshThreads) filter_hist_kernel(FilterArgs a, int pass) {
    __shared__ uint32_t h[256];
    static_assert(kMeshThreads == 256, "one bin per thread");
    h[threadIdx.x] = 0;
    __syncthreads();
    const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (t < a.Nt && a.sel[1] && a.label[t] == (uint32_t)t) {
        const int shift = 24 - 8 * pass;
        const uint32_t s = a.size[t], high = pass ? ~0u << (shift + 8) : 0u;
        if ((s & high) == (a.sel[0] & high)) atomicAdd(h + ((s >> shift) & 255), 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(a.hist + 256 * pass + threadIdx.x, h[threadIdx.x]);
}

// keep flags over the labels, and idempotent used marks of the kept triangles' vertices
__global__ void __launch_bounds__(kMeshThreads) filter_keep_kernel(FilterArgs a) {
    const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (t >= a.Nt) return;
    const uint32_t r = a.label[t];
    const bool kept = r != kDead && a.size[r] >= a.sel[0];
    a.label[t] = kept ? 1u : 0u;
    if (kept) {
        const int32_t* tri = a.triangles + 3 * (size_t)t;
        a.used[__ldg(tri)] = 1u;
        a.used[__ldg(tri + 1)] = 1u;
        a.used[__ldg(tri + 2)] = 1u;
    }
}

struct FilterEmitArgs {
    int Nv, Nt, Nv_out, Nt_out;
    const float* vertices; const float* colors; const int32_t* triangles;
    const uint32_t* label; const uint32_t* used;
    float* out_vertices; float* out_colors; int32_t* out_triangles;
};

// one thread per vertex and per triangle (the same index), each written at its scanned offset
__global__ void __launch_bounds__(kMeshThreads) filter_emit_kernel(FilterEmitArgs a) {
    const long long i = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
    if (i < a.Nv) {
        const uint32_t o = a.used[i];
        if (a.used[i + 1] != o && o < (uint32_t)a.Nv_out) {
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                a.out_vertices[3 * (size_t)o + r] = __ldg(a.vertices + 3 * (size_t)i + r);
                a.out_colors[3 * (size_t)o + r] = __ldg(a.colors + 3 * (size_t)i + r);
            }
        }
    }
    if (i < a.Nt) {
        const uint32_t o = a.label[i];
        if (a.label[i + 1] != o && o < (uint32_t)a.Nt_out) {
#pragma unroll
            for (int m = 0; m < 3; ++m) {
                const int32_t v = __ldg(a.triangles + 3 * (size_t)i + m);
                a.out_triangles[3 * (size_t)o + m] = (uint32_t)v < (uint32_t)a.Nv ? (int32_t)a.used[v] : -1;
            }
        }
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

extern "C" int srf_mesh_filter_workspace_bytes(int Nv, int Nt, size_t* bytes) {
    if (Nv < 0 || Nt < 0) return set_error("srf_mesh_filter_workspace_bytes: bad sizes (Nv=%d, Nt=%d)", Nv, Nt);
    if (!bytes) return set_error("srf_mesh_filter_workspace_bytes: null output");
    *bytes = srf::filter_layout((size_t)Nv, (size_t)Nt).total;
    return 0;
}

extern "C" int srf_mesh_filter_count(void* stream_, int Nv, int Nt, const float* vertices, const int32_t* triangles,
                                     const double* aabb, int keep, void* workspace, int32_t* totals) {
    const char* fn = "srf_mesh_filter_count";
    if (Nv < 0 || Nt < 0) return set_error("%s: bad sizes (Nv=%d, Nt=%d)", fn, Nv, Nt);
    if (keep < 1) return set_error("%s: keep must be >= 1, got %d", fn, keep);
    if ((Nv > 0 && !vertices) || (Nt > 0 && !triangles) || !totals) return set_error("%s: null pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const cudaStream_t stream = (cudaStream_t)stream_;
    const srf::FilterWorkspace l = srf::filter_layout((size_t)Nv, (size_t)Nt);
    char* ws = static_cast<char*>(workspace);
    srf::FilterArgs a;
    a.Nv = Nv; a.Nt = Nt; a.keep = keep; a.crop = aabb != nullptr;
    for (int r = 0; r < 3; ++r) {
        a.lo[r] = aabb ? aabb[r] : 0.0;
        a.hi[r] = aabb ? aabb[3 + r] : 0.0;
    }
    a.mask = l.slots - 1;
    a.vertices = vertices; a.triangles = triangles;
    a.keys = reinterpret_cast<unsigned long long*>(ws + l.keys);
    a.owner = reinterpret_cast<uint32_t*>(ws + l.owner);
    a.parent = reinterpret_cast<int32_t*>(ws + l.parent);
    a.size = reinterpret_cast<uint32_t*>(ws + l.size);
    a.label = reinterpret_cast<uint32_t*>(ws + l.label);
    a.used = reinterpret_cast<uint32_t*>(ws + l.used);
    a.hist = reinterpret_cast<uint32_t*>(ws + l.hist);
    a.sel = reinterpret_cast<uint32_t*>(ws + l.sel);
    a.totals = totals;
    uint32_t* sums = reinterpret_cast<uint32_t*>(ws + l.sums);
    cudaError_t e;
    if ((e = cudaMemsetAsync(totals, 0, 4 * sizeof(int32_t), stream)) != cudaSuccess ||
        (e = cudaMemsetAsync(a.used, 0, 4 * (size_t)Nv, stream)) != cudaSuccess)
        return cuda_error("memset mesh filter totals", e);
    if (Nt > 0) {
        if ((e = cudaMemsetAsync(a.keys, 0xff, 8 * l.slots, stream)) != cudaSuccess ||
            (e = cudaMemsetAsync(a.owner, 0xff, 4 * l.slots, stream)) != cudaSuccess ||
            (e = cudaMemsetAsync(a.size, 0, 4 * (size_t)Nt, stream)) != cudaSuccess ||
            (e = cudaMemsetAsync(a.hist, 0, 4 * 256 * srf::kSelectPasses, stream)) != cudaSuccess)
            return cuda_error("memset mesh filter workspace", e);
        const unsigned blocks = (unsigned)(((size_t)Nt + srf::kMeshThreads - 1) / srf::kMeshThreads);
        srf::filter_crop_kernel<<<blocks, srf::kMeshThreads, 0, stream>>>(a);
        srf::filter_insert_kernel<<<blocks, srf::kMeshThreads, 0, stream>>>(a);
        srf::filter_union_kernel<<<blocks, srf::kMeshThreads, 0, stream>>>(a);
        srf::filter_label_kernel<<<blocks, srf::kMeshThreads, 0, stream>>>(a);
        srf::filter_select_kernel<<<1, 1, 0, stream>>>(a, -1);
        for (int pass = 0; pass < srf::kSelectPasses; ++pass) {
            srf::filter_hist_kernel<<<blocks, srf::kMeshThreads, 0, stream>>>(a, pass);
            srf::filter_select_kernel<<<1, 1, 0, stream>>>(a, pass);
        }
        srf::filter_keep_kernel<<<blocks, srf::kMeshThreads, 0, stream>>>(a);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error("mesh filter launch", e);
    }
    // with Nt = 0 the label flags are empty and the used flags all 0: the scans write the totals 0
    if ((e = srf::exclusive_scan(a.used, (size_t)Nv, sums + l.nb_tri, l.nb_vert, totals, stream)) != cudaSuccess ||
        (e = srf::exclusive_scan(a.label, (size_t)Nt, sums, l.nb_tri, totals + 1, stream)) != cudaSuccess)
        return cuda_error("mesh filter scan launch", e);
    return 0;
}

extern "C" int srf_mesh_filter_emit(void* stream, int Nv, int Nt, const float* vertices, const float* colors,
                                    const int32_t* triangles, const void* workspace, int Nv_out, int Nt_out,
                                    float* out_vertices, float* out_colors, int32_t* out_triangles) {
    const char* fn = "srf_mesh_filter_emit";
    if (Nv < 0 || Nt < 0) return set_error("%s: bad sizes (Nv=%d, Nt=%d)", fn, Nv, Nt);
    if (Nv_out < 0 || Nt_out < 0 || Nv_out > Nv || Nt_out > Nt)
        return set_error("%s: bad totals (Nv_out=%d, Nt_out=%d for Nv=%d, Nt=%d)", fn, Nv_out, Nt_out, Nv, Nt);
    if ((Nv > 0 && (!vertices || !colors)) || (Nt > 0 && !triangles)) return set_error("%s: null input pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    if ((Nv_out > 0 && (!out_vertices || !out_colors)) || (Nt_out > 0 && !out_triangles))
        return set_error("%s: null output pointer", fn);
    if (Nv_out == 0 && Nt_out == 0) return 0;
    const srf::FilterWorkspace l = srf::filter_layout((size_t)Nv, (size_t)Nt);
    const char* ws = static_cast<const char*>(workspace);
    srf::FilterEmitArgs a;
    a.Nv = Nv; a.Nt = Nt; a.Nv_out = Nv_out; a.Nt_out = Nt_out;
    a.vertices = vertices; a.colors = colors; a.triangles = triangles;
    a.label = reinterpret_cast<const uint32_t*>(ws + l.label);
    a.used = reinterpret_cast<const uint32_t*>(ws + l.used);
    a.out_vertices = out_vertices; a.out_colors = out_colors; a.out_triangles = out_triangles;
    const size_t n = (size_t)(Nv > Nt ? Nv : Nt);
    const unsigned blocks = (unsigned)((n + srf::kMeshThreads - 1) / srf::kMeshThreads);
    srf::filter_emit_kernel<<<blocks, srf::kMeshThreads, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("mesh_filter_emit launch", e);
}
