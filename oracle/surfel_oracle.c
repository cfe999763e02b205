/* surfel_oracle.c -- CPU restatement of the reference rasterizer's algorithm.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may build, load or call this file.  The product
 * (lara_b200/) never does and has no CPU fallback.
 *
 * Parity pinning: the reference (LaRa third_party/diff-surfel-rasterization, "DSR")
 * ships no tests, fixtures or golden vectors for this path (SURVEY.md 8c).  This oracle is
 * therefore pinned against golden input/output vectors produced by running the reference's
 * own sm_100 CUDA build on a B200: tests/golden/ + tests/golden/make_golden.py.
 *
 * Plain C, fp32 with fmaf() placed exactly where nvcc fused the reference's expressions
 * (compile with -ffp-contract=off), so everything except rsqrt/exp (approximate units on
 * the GPU) reproduces the reference bit for bit.  Each function cites the reference
 * file:line it restates (paths relative to DSR/cuda_rasterizer/).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE 16
#define NEAR_F 0.2f

typedef struct {
    int P, D, M, H, W;
    float tanfovx, tanfovy;
    const float* bg;            /* [3] */
    const float* means3D;       /* [P,3] */
    const float* shs;           /* [P,M,3] or NULL */
    const float* colors_precomp;/* [P,3] or NULL */
    const float* opacities;     /* [P] */
    const float* scales;        /* [P,2] */
    const float* rotations;     /* [P,4] wxyz */
    const float* viewmatrix;    /* [16] column-major */
    const float* campos;        /* [3] */
} OracleIn;

typedef struct {
    OracleIn in;
    int gx, gy, ntiles;
    float focal_x, focal_y;
    /* per Gaussian (rasterizer_impl.cu:155-170 GeometryState) */
    int* radii;
    float* depths;
    float* T;        /* [P,9] */
    float* center;   /* [P,2] */
    float* normal;   /* [P,3] */
    float* rgb;      /* [P,3] */
    uint8_t* clamped;/* [P,3] */
    uint32_t* rect;  /* [P,4] x0,y0,x1,y1 */
    uint32_t* tiles_touched;
    /* binning (rasterizer_impl.cu:181-194) */
    uint32_t num_rendered;
    uint64_t* keys;      /* sorted */
    uint32_t* point_list;/* sorted */
    uint32_t* ranges;    /* [ntiles,2] */
    /* image state (rasterizer_impl.cu:172-179) */
    float* accum;        /* [3,H,W] final_T, dist1, dist2 */
    uint32_t* n_contrib; /* [2,H,W] */
    float* out_color;    /* [3,H,W] */
    float* out_others;   /* [8,H,W] */
    uint32_t* masks;     /* [8, num_rendered] contribution record, the kernels' layout: bit l of block w = pixel
                            (col (w&1)*8 + (l&7), row (w>>1)*4 + (l>>3)) of the tile blended list position j */
} Oracle;

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }
static inline int f2i(float x) { /* cvt.rzi.s32.f32: truncate, saturate, NaN -> 0 */
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return (int)0x80000000;
    return (int)x;
}

/* quaternion -> rotation columns (auxiliary.h:188-210); the reference uses rsqrtf */
static void quat_to_R(const float* q, float R[3][3]) {
    const float n2 = fmaf(q[2], q[2], fmaf(q[1], q[1], fmaf(q[3], q[3], q[0] * q[0])));
    const float s = 1.0f / sqrtf(n2);
    const float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
    const float wz = w * z, wy = w * y, wx = w * x, yy = y * y, zz = z * z;
    const float xy_p = fmaf(x, y, wz), xy_m = fmaf(x, y, -wz);
    const float yz_p = fmaf(y, z, wx), yz_m = fmaf(y, z, -wx);
    const float xz_m = fmaf(x, z, -wy), xz_p = fmaf(x, z, wy);
    const float yyzz = yy + zz, xxzz = fmaf(x, x, zz), xxyy = fmaf(x, x, yy);
    R[0][0] = 1.0f - (yyzz + yyzz); R[0][1] = xy_p + xy_p; R[0][2] = xz_m + xz_m;
    R[1][0] = xy_m + xy_m; R[1][1] = 1.0f - (xxzz + xxzz); R[1][2] = yz_p + yz_p;
    R[2][0] = xz_p + xz_p; R[2][1] = yz_m + yz_m; R[2][2] = 1.0f - (xxyy + xxyy);
}

/* W * v for the column-major view rotation, in the fused order of the reference build */
static inline float wdot(float a, float b, float c, float x, float y, float z) {
    return fmaf(c, z, fmaf(a, x, b * y));
}

/* SH -> RGB (forward.cu:20-71) */
static void sh_to_rgb(int deg, const float* sh, const float dir[3], float rgb[3]) {
    const float x = dir[0], y = dir[1], z = dir[2];
    for (int c = 0; c < 3; ++c) {
        float r = SH_C0 * sh[c];
        if (deg > 0) {
            r = r - SH_C1 * y * sh[3 + c] + SH_C1 * z * sh[6 + c] - SH_C1 * x * sh[9 + c];
            if (deg > 1) {
                const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                r = r + SH_C2[0] * xy * sh[12 + c] + SH_C2[1] * yz * sh[15 + c] +
                    SH_C2[2] * (2.0f * zz - xx - yy) * sh[18 + c] + SH_C2[3] * xz * sh[21 + c] +
                    SH_C2[4] * (xx - yy) * sh[24 + c];
                if (deg > 2) {
                    r = r + SH_C3[0] * y * (3.0f * xx - yy) * sh[27 + c] + SH_C3[1] * xy * z * sh[30 + c] +
                        SH_C3[2] * y * (4.0f * zz - xx - yy) * sh[33 + c] +
                        SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[36 + c] +
                        SH_C3[4] * x * (4.0f * zz - xx - yy) * sh[39 + c] + SH_C3[5] * z * (xx - yy) * sh[42 + c] +
                        SH_C3[6] * x * (xx - 3.0f * yy) * sh[45 + c];
                }
            }
        }
        rgb[c] = r + 0.5f;
    }
}

/* K1: forward.cu:166-260 with auxiliary.h:160-185 (cull), forward.cu:75-128 (T),
 * :133-163 (AABB), :237-259 + auxiliary.h:64-74 (radius, rect). */
static void preprocess_one(Oracle* o, int i) {
    const OracleIn* in = &o->in;
    const float* v = in->viewmatrix;
    const float px = in->means3D[3 * i], py = in->means3D[3 * i + 1], pz = in->means3D[3 * i + 2];
    o->radii[i] = 0; o->tiles_touched[i] = 0;
    o->rect[4 * i] = o->rect[4 * i + 1] = o->rect[4 * i + 2] = o->rect[4 * i + 3] = 0;
    const float pvz = fmaf(pz, v[10], fmaf(px, v[2], py * v[6])) + v[14];
    if (pvz <= 0.2f) return;
    float R[3][3];
    quat_to_R(in->rotations + 4 * i, R);
    const float sx = in->scales[2 * i], sy = in->scales[2 * i + 1];
    const float a0[3] = {R[0][0] * sx, R[0][1] * sx, R[0][2] * sx};
    const float a1[3] = {R[1][0] * sy, R[1][1] * sy, R[1][2] * sy};
    const float pvx = v[12] + fmaf(pz, v[8], fmaf(px, v[0], py * v[4]));
    const float pvy = v[13] + fmaf(pz, v[9], fmaf(px, v[1], py * v[5]));
    const float tnx = wdot(v[0], v[4], v[8], R[2][0], R[2][1], R[2][2]);
    const float tny = wdot(v[1], v[5], v[9], R[2][0], R[2][1], R[2][2]);
    const float tnz = wdot(v[2], v[6], v[10], R[2][0], R[2][1], R[2][2]);
    const float cosv = fmaf(-pvz, tnz, fmaf(pvy, -tny, -(pvx * tnx)));
    if (cosv == 0.0f) return;
    const float M0x = wdot(v[0], v[4], v[8], a0[0], a0[1], a0[2]);
    const float M0y = wdot(v[1], v[5], v[9], a0[0], a0[1], a0[2]);
    const float M0z = wdot(v[2], v[6], v[10], a0[0], a0[1], a0[2]);
    const float M1x = wdot(v[0], v[4], v[8], a1[0], a1[1], a1[2]);
    const float M1y = wdot(v[1], v[5], v[9], a1[0], a1[1], a1[2]);
    const float M1z = wdot(v[2], v[6], v[10], a1[0], a1[1], a1[2]);
    const float cxh = (float)in->W * 0.5f, cyh = (float)in->H * 0.5f;
    float* T = o->T + 9 * i;
    T[0] = fmaf(M0z, cxh, M0x * o->focal_x); T[1] = fmaf(M1z, cxh, M1x * o->focal_x); T[2] = fmaf(pvz, cxh, pvx * o->focal_x);
    T[3] = fmaf(M0z, cyh, M0y * o->focal_y); T[4] = fmaf(M1z, cyh, M1y * o->focal_y); T[5] = fmaf(pvz, cyh, pvy * o->focal_y);
    T[6] = M0z; T[7] = M1z; T[8] = pvz;
    const float mult = cosv > 0.0f ? 1.0f : -1.0f;
    const float d = fmaf(-T[8], T[8], fmaf(T[6], T[6], T[7] * T[7]));
    if (d == 0.0f) return;
    const float inv = 1.0f / d;
    float t = (T[0] * T[6]) * inv;
    t = fmaf(T[1] * T[7], inv, t);
    const float cx = fmaf(T[2] * T[8], -inv, t);
    float b = (T[0] * T[0]) * inv;
    b = fmaf(T[1] * T[1], inv, b);
    const float h0x = fmaf(cx, cx, fmaf(T[2] * T[2], inv, -b));
    t = (T[3] * T[6]) * inv;
    t = fmaf(T[4] * T[7], inv, t);
    const float cy = fmaf(T[5] * T[8], -inv, t);
    b = (T[3] * T[3]) * inv;
    b = fmaf(T[4] * T[4], inv, b);
    const float h0y = fmaf(cy, cy, fmaf(T[5] * T[5], inv, -b));
    const float ex = sqrtf(fmaxf(0.0f, h0x)), ey = sqrtf(fmaxf(0.0f, h0y));
    const float e = fmaxf(ex, ey);
    const double rd = ceil(3.0 * fmax((double)e, 0.7071067811865476));
    const int radius = f2i((float)rd);
    const float rf = (float)radius;
    const int x0 = imin(o->gx, imax(0, f2i((cx - rf) * 0.0625f)));
    const int y0 = imin(o->gy, imax(0, f2i((cy - rf) * 0.0625f)));
    const int x1 = imin(o->gx, imax(0, f2i((((cx + rf) + 16.0f) - 1.0f) * 0.0625f)));
    const int y1 = imin(o->gy, imax(0, f2i((((cy + rf) + 16.0f) - 1.0f) * 0.0625f)));
    if ((x1 - x0) * (y1 - y0) == 0) return;
    if (in->colors_precomp == NULL) {
        float dir[3] = {px - in->campos[0], py - in->campos[1], pz - in->campos[2]};
        const float len = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        dir[0] /= len; dir[1] /= len; dir[2] /= len;
        float rgb[3];
        sh_to_rgb(in->D, in->shs + (size_t)i * 3 * in->M, dir, rgb);
        for (int c = 0; c < 3; ++c) {
            o->clamped[3 * i + c] = rgb[c] < 0.0f;
            o->rgb[3 * i + c] = fmaxf(rgb[c], 0.0f);
        }
    } else {
        for (int c = 0; c < 3; ++c) { o->rgb[3 * i + c] = in->colors_precomp[3 * i + c]; o->clamped[3 * i + c] = 0; }
    }
    o->depths[i] = pvz;
    o->radii[i] = radius;
    o->center[2 * i] = cx; o->center[2 * i + 1] = cy;
    o->normal[3 * i] = tnx * mult; o->normal[3 * i + 1] = tny * mult; o->normal[3 * i + 2] = tnz * mult;
    o->rect[4 * i] = x0; o->rect[4 * i + 1] = y0; o->rect[4 * i + 2] = x1; o->rect[4 * i + 3] = y1;
    o->tiles_touched[i] = (uint32_t)((x1 - x0) * (y1 - y0));
}

typedef struct { uint64_t key; uint32_t val; } KV;
static int kv_cmp(const void* a, const void* b) {
    const KV* x = (const KV*)a; const KV* y = (const KV*)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->val < y->val ? -1 : (x->val > y->val);   /* stable sort == ascending emission order */
}

/* K2-K5: rasterizer_impl.cu:70-111 (keys), :301-309 (sort), :116-138 (ranges) */
static int bin_and_sort(Oracle* o) {
    const int P = o->in.P;
    uint64_t R = 0;
    for (int i = 0; i < P; ++i) R += o->tiles_touched[i];
    o->num_rendered = (uint32_t)R;
    KV* kv = (KV*)malloc((R ? R : 1) * sizeof(KV));
    if (!kv) return 1;
    uint64_t off = 0;
    for (int i = 0; i < P; ++i) {
        if (o->radii[i] <= 0) continue;
        uint32_t dbits; memcpy(&dbits, &o->depths[i], 4);
        for (uint32_t y = o->rect[4 * i + 1]; y < o->rect[4 * i + 3]; ++y)
            for (uint32_t x = o->rect[4 * i]; x < o->rect[4 * i + 2]; ++x) {
                kv[off].key = ((uint64_t)(y * (uint32_t)o->gx + x) << 32) | dbits;
                kv[off].val = (uint32_t)i;
                ++off;
            }
    }
    qsort(kv, R, sizeof(KV), kv_cmp);
    o->keys = (uint64_t*)malloc((R ? R : 1) * sizeof(uint64_t));
    o->point_list = (uint32_t*)malloc((R ? R : 1) * sizeof(uint32_t));
    o->masks = (uint32_t*)calloc((R ? R : 1) * 8, sizeof(uint32_t));
    for (uint64_t j = 0; j < R; ++j) { o->keys[j] = kv[j].key; o->point_list[j] = kv[j].val; }
    free(kv);
    memset(o->ranges, 0, (size_t)o->ntiles * 2 * sizeof(uint32_t));
    for (uint64_t j = 0; j < R; ++j) {
        const uint32_t t = (uint32_t)(o->keys[j] >> 32);
        if (j == 0 || t != (uint32_t)(o->keys[j - 1] >> 32)) {
            o->ranges[2 * t] = (uint32_t)j;
            if (j) o->ranges[2 * (o->keys[j - 1] >> 32) + 1] = (uint32_t)j;
        }
        if (j == R - 1) o->ranges[2 * t + 1] = (uint32_t)R;
    }
    return 0;
}

/* the per-(pixel,splat) evaluation shared by forward and backward
 * (forward.cu:353-398, backward.cu:258-318) */
typedef struct {
    float kx, ky, kz, lx, ly, lz, px, py, pz, sx, sy, dx, dy, rho3d, rho2d, depth, G, alpha;
} Pair;

/* the two footprints of a pair, rho3d and rho2d; returns 0 where p.z == 0 */
static int pair_footprints(const float* T, const float* center, float pixx, float pixy, Pair* e) {
    e->kx = fmaf(pixx, T[6], -T[0]); e->ky = fmaf(pixx, T[7], -T[1]); e->kz = fmaf(pixx, T[8], -T[2]);
    e->lx = fmaf(pixy, T[6], -T[3]); e->ly = fmaf(pixy, T[7], -T[4]); e->lz = fmaf(pixy, T[8], -T[5]);
    e->pz = fmaf(e->kx, e->ly, -(e->ky * e->lx));
    e->px = fmaf(e->ky, e->lz, -(e->kz * e->ly));
    e->py = fmaf(e->kz, e->lx, -(e->kx * e->lz));
    if (e->pz == 0.0f) return 0;
    e->sx = e->px / e->pz; e->sy = e->py / e->pz;
    e->rho3d = fmaf(e->sx, e->sx, e->sy * e->sy);
    e->dx = center[0] - pixx; e->dy = center[1] - pixy;
    /* (float)(FilterInvSquare(double) * (double)|d|^2), FilterInvSquare = 1/(0.7071..^2) (auxiliary.h:20-21) */
    e->rho2d = (float)((1 / (0.7071067811865476 * 0.7071067811865476)) * (double)fmaf(e->dx, e->dx, e->dy * e->dy));
    return 1;
}

static int eval_pair(const Oracle* o, uint32_t g, float pixx, float pixy, Pair* e) {
    const float* T = o->T + 9 * (size_t)g;
    if (!pair_footprints(T, o->center + 2 * (size_t)g, pixx, pixy, e)) return 0;
    const float rho = fminf(e->rho3d, e->rho2d);
    e->depth = (e->rho3d <= e->rho2d) ? (T[8] + fmaf(T[6], e->sx, T[7] * e->sy)) : T[8];
    if ((double)e->depth < 0.2) return 0;
    const float power = -0.5f * rho;
    if (power > 0.0f) return 0;
    e->G = expf(power);
    e->alpha = fminf(0.99f, o->in.opacities[g] * e->G);
    if (e->alpha < 1.0f / 255.0f) return 0;
    return 1;
}

/* K6: forward.cu:265-463 */
static void blend_forward(Oracle* o) {
    const int H = o->in.H, W = o->in.W;
    const size_t npix = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < o->ntiles; ++tile) {
        const int ty = tile / o->gx, tx = tile % o->gx;
        const uint32_t r0 = o->ranges[2 * tile], r1 = o->ranges[2 * tile + 1];
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            const float pixx = (float)x + 0.5f, pixy = (float)y + 0.5f;
            float Tr = 1.0f, C[3] = {0, 0, 0}, N[3] = {0, 0, 0};
            float D = 0, dist1 = 0, dist2 = 0, distortion = 0, med_d = 0, med_w = 0, med_c = -1.0f;
            uint32_t contributor = 0, last = 0;
            for (uint32_t j = r0; j < r1; ++j) {
                contributor++;
                const uint32_t g = o->point_list[j];
                Pair e;
                if (!eval_pair(o, g, pixx, pixy, &e)) continue;
                const float alpha = e.alpha;
                const float test_T = Tr * (1.0f - alpha);
                if (test_T < 0.0001f) break;
                const float A = 1.0f - Tr;
                const double dd = (double)e.depth;
                const float m = (float)((100.0 * dd - 100.0 * 0.2) / ((100.0 - 0.2) * dd));
                const float mm = m * m;
                const float err = fmaf(-dist1, m + m, fmaf(A, mm, dist2));
                distortion = fmaf(Tr, alpha * err, distortion);
                if (Tr > 0.5f) { med_d = e.depth; med_w = Tr * alpha; med_c = (float)contributor; }
                for (int c = 0; c < 3; ++c) N[c] = fmaf(Tr, o->normal[3 * (size_t)g + c] * alpha, N[c]);
                D = fmaf(Tr, e.depth * alpha, D);
                dist1 = fmaf(Tr, alpha * m, dist1);
                dist2 = fmaf(Tr, alpha * mm, dist2);
                for (int c = 0; c < 3; ++c) C[c] = fmaf(Tr, alpha * o->rgb[3 * (size_t)g + c], C[c]);
                Tr = test_T;
                last = contributor;
                o->masks[(size_t)((ly >> 2) * 2 + (lx >> 3)) * o->num_rendered + j] |= 1u << ((ly & 3) * 8 + (lx & 7));
            }
            const size_t pix = (size_t)y * W + x;
            o->accum[pix] = Tr; o->accum[pix + npix] = dist1; o->accum[pix + 2 * npix] = dist2;
            o->n_contrib[pix] = last;
            o->n_contrib[pix + npix] = med_c < 0.0f ? 0u : (uint32_t)med_c;
            for (int c = 0; c < 3; ++c) o->out_color[pix + c * npix] = fmaf(o->in.bg[c], Tr, C[c]);
            o->out_others[pix] = D;
            o->out_others[pix + npix] = 1.0f - Tr;
            for (int c = 0; c < 3; ++c) o->out_others[pix + (2 + c) * npix] = N[c];
            o->out_others[pix + 5 * npix] = med_d;
            o->out_others[pix + 6 * npix] = distortion;
            o->out_others[pix + 7 * npix] = med_w;
        }
    }
}

void oracle_destroy(Oracle* o) {
    if (!o) return;
    free(o->radii); free(o->depths); free(o->T); free(o->center); free(o->normal); free(o->rgb);
    free(o->clamped); free(o->rect); free(o->tiles_touched); free(o->keys); free(o->point_list); free(o->masks);
    free(o->ranges); free(o->accum); free(o->n_contrib); free(o->out_color); free(o->out_others);
    free(o);
}

/* Rasterizer::forward (rasterizer_impl.cu:198-342).  The caller keeps the input arrays alive. */
Oracle* oracle_forward(const OracleIn* in) {
    Oracle* o = (Oracle*)calloc(1, sizeof(Oracle));
    if (!o) return NULL;
    o->in = *in;
    const int P = in->P, H = in->H, W = in->W;
    o->gx = (W + TILE - 1) / TILE; o->gy = (H + TILE - 1) / TILE; o->ntiles = o->gx * o->gy;
    o->focal_y = H / (2.0f * in->tanfovy);
    o->focal_x = W / (2.0f * in->tanfovx);
    const size_t p = P > 0 ? (size_t)P : 1, npix = (size_t)H * W;
    o->radii = (int*)calloc(p, sizeof(int));
    o->depths = (float*)calloc(p, sizeof(float));
    o->T = (float*)calloc(p * 9, sizeof(float));
    o->center = (float*)calloc(p * 2, sizeof(float));
    o->normal = (float*)calloc(p * 3, sizeof(float));
    o->rgb = (float*)calloc(p * 3, sizeof(float));
    o->clamped = (uint8_t*)calloc(p * 3, 1);
    o->rect = (uint32_t*)calloc(p * 4, sizeof(uint32_t));
    o->tiles_touched = (uint32_t*)calloc(p, sizeof(uint32_t));
    o->ranges = (uint32_t*)calloc((size_t)o->ntiles * 2, sizeof(uint32_t));
    o->accum = (float*)calloc(npix * 3, sizeof(float));
    o->n_contrib = (uint32_t*)calloc(npix * 2, sizeof(uint32_t));
    o->out_color = (float*)calloc(npix * 3, sizeof(float));
    o->out_others = (float*)calloc(npix * 8, sizeof(float));
    if (P == 0) return o;   /* rasterize_points.cu:105: nothing runs, outputs stay zero */
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; ++i) preprocess_one(o, i);
    if (bin_and_sort(o)) { oracle_destroy(o); return NULL; }
    blend_forward(o);
    return o;
}

static inline void atomic_add_d(double* p, double v) {
#pragma omp atomic
    *p += v;
}

/* K7: backward.cu:143-449.  Per-Gaussian partials are summed in double (the reference uses
 * fp32 atomics in nondeterministic order; double is the value both GPU versions approximate). */
static void blend_backward(const Oracle* o, const float* dL_dpix, const float* dL_dothers,
                           double* dT, double* dmean2D, double* dnormal, double* dopac, double* dcolor) {
    const int H = o->in.H, W = o->in.W;
    const size_t npix = (size_t)H * W;
    const float* bg = o->in.bg;
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < o->ntiles; ++tile) {
        const int ty = tile / o->gx, tx = tile % o->gx;
        const uint32_t r0 = o->ranges[2 * tile];
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            const size_t pix = (size_t)y * W + x;
            const float pixx = (float)x + 0.5f, pixy = (float)y + 0.5f;
            const float T_final = o->accum[pix];
            float Tr = T_final;
            const int last_contributor = (int)o->n_contrib[pix];
            const int median_contributor = (int)o->n_contrib[pix + npix];
            const float dpix[3] = {dL_dpix[pix], dL_dpix[pix + npix], dL_dpix[pix + 2 * npix]};
            const float dL_ddepth = dL_dothers[pix], dL_daccum = dL_dothers[pix + npix];
            const float dn[3] = {dL_dothers[pix + 2 * npix], dL_dothers[pix + 3 * npix], dL_dothers[pix + 4 * npix]};
            const float dL_dmedian_depth = dL_dothers[pix + 5 * npix], dL_dreg = dL_dothers[pix + 6 * npix];
            const float dL_dmax_dweight = dL_dothers[pix + 7 * npix];
            const float final_D = o->accum[pix + npix], final_D2 = o->accum[pix + 2 * npix];
            const float final_A = 1.0f - T_final;
            float accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_normal[3] = {0, 0, 0}, accum_normal_rec[3] = {0, 0, 0};
            float last_alpha = 0, last_depth = 0, accum_depth_rec = 0, accum_alpha_rec = 0, last_dL_dT = 0;
            float bg_dot = 0;
            for (int c = 0; c < 3; ++c) bg_dot += bg[c] * dpix[c];
            for (int pos = last_contributor - 1; pos >= 0; --pos) {
                const uint32_t g = o->point_list[r0 + (uint32_t)pos];
                Pair e;
                if (!eval_pair(o, g, pixx, pixy, &e)) continue;
                const float alpha = e.alpha, G = e.G, c_d = e.depth;
                const float* T = o->T + 9 * (size_t)g;
                Tr = Tr / (1.0f - alpha);
                const float w = alpha * Tr;
                float dL_dalpha = 0.0f;
                for (int c = 0; c < 3; ++c) {
                    const float col = o->rgb[3 * (size_t)g + c];
                    accum_rec[c] = last_alpha * last_color[c] + (1.f - last_alpha) * accum_rec[c];
                    last_color[c] = col;
                    dL_dalpha += (col - accum_rec[c]) * dpix[c];
                    atomic_add_d(&dcolor[3 * (size_t)g + c], (double)(w * dpix[c]));
                }
                float dL_dz = 0.0f, dL_dweight = 0.0f;
                const double cd = (double)c_d;
                const float m_d = (float)((100.0 * cd - 100.0 * 0.2) / ((100.0 - 0.2) * cd));
                const float dmd_dd = (float)((100.0 * 0.2) / ((100.0 - 0.2) * cd * cd));
                if (pos == median_contributor - 1) { dL_dz += dL_dmedian_depth; dL_dweight += dL_dmax_dweight; }
                dL_dweight += (final_D2 + m_d * m_d * final_A - 2 * m_d * final_D) * dL_dreg;
                dL_dalpha += dL_dweight - last_dL_dT;
                last_dL_dT = dL_dweight * alpha + (1 - alpha) * last_dL_dT;
                const float dL_dmd = 2.0f * (Tr * alpha) * (m_d * final_A - final_D) * dL_dreg;
                dL_dz += dL_dmd * dmd_dd;
                accum_depth_rec = last_alpha * last_depth + (1.f - last_alpha) * accum_depth_rec;
                last_depth = c_d;
                dL_dalpha += (c_d - accum_depth_rec) * dL_ddepth;
                accum_alpha_rec = last_alpha * 1.0f + (1.f - last_alpha) * accum_alpha_rec;
                dL_dalpha += (1 - accum_alpha_rec) * dL_daccum;
                for (int c = 0; c < 3; ++c) {
                    const float nc = o->normal[3 * (size_t)g + c];
                    accum_normal_rec[c] = last_alpha * last_normal[c] + (1.f - last_alpha) * accum_normal_rec[c];
                    last_normal[c] = nc;
                    dL_dalpha += (nc - accum_normal_rec[c]) * dn[c];
                    atomic_add_d(&dnormal[3 * (size_t)g + c], (double)(w * dn[c]));
                }
                dL_dalpha *= Tr;
                last_alpha = alpha;
                dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
                const float dL_dG = o->in.opacities[g] * dL_dalpha;
                dL_dz += w * dL_ddepth;
                if (e.rho3d <= e.rho2d) {
                    const float dsx = dL_dG * -G * e.sx + dL_dz * T[6];
                    const float dsy = dL_dG * -G * e.sy + dL_dz * T[7];
                    const float dsx_pz = dsx / e.pz, dsy_pz = dsy / e.pz;
                    const float dp[3] = {dsx_pz, dsy_pz, -(dsx_pz * e.sx + dsy_pz * e.sy)};
                    const float dk[3] = {e.ly * dp[2] - e.lz * dp[1], e.lz * dp[0] - e.lx * dp[2], e.lx * dp[1] - e.ly * dp[0]};
                    const float dl[3] = {dp[1] * e.kz - dp[2] * e.ky, dp[2] * e.kx - dp[0] * e.kz, dp[0] * e.ky - dp[1] * e.kx};
                    const float dz_dTw[3] = {e.sx, e.sy, 1.0f};
                    for (int c = 0; c < 3; ++c) {
                        atomic_add_d(&dT[9 * (size_t)g + c], (double)(-dk[c]));
                        atomic_add_d(&dT[9 * (size_t)g + 3 + c], (double)(-dl[c]));
                        atomic_add_d(&dT[9 * (size_t)g + 6 + c], (double)(pixx * dk[c] + pixy * dl[c] + dL_dz * dz_dTw[c]));
                    }
                } else {
                    const float dG_ddelx = (float)(-G * (1 / (0.7071067811865476 * 0.7071067811865476)) * e.dx);
                    const float dG_ddely = (float)(-G * (1 / (0.7071067811865476 * 0.7071067811865476)) * e.dy);
                    atomic_add_d(&dmean2D[2 * (size_t)g], (double)(dL_dG * dG_ddelx));
                    atomic_add_d(&dmean2D[2 * (size_t)g + 1], (double)(dL_dG * dG_ddely));
                    atomic_add_d(&dT[9 * (size_t)g + 8], (double)dL_dz);
                }
                atomic_add_d(&dopac[g], (double)(G * dL_dalpha));
            }
        }
    }
}

/* K8 + K9: backward.cu:599-649, :533-597, :451-529, :20-139, auxiliary.h:213-257,125-135 */
static void preprocess_backward_one(const Oracle* o, int i, const double* dTd, const double* dm2, const double* dnrm,
                                    const double* dcol, float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh,
                                    float* dL_dscales, float* dL_drot, float* dL_dtransMat) {
    const OracleIn* in = &o->in;
    if (!(o->radii[i] > 0)) return;
    const float* T = o->T + 9 * (size_t)i;
    float dT[9];
    for (int k = 0; k < 9; ++k) dT[k] = (float)dTd[9 * (size_t)i + k];
    const float dmx = (float)dm2[2 * (size_t)i], dmy = (float)dm2[2 * (size_t)i + 1];
    {   /* computeAABB backward */
        const float d = T[6] * T[6] + T[7] * T[7] - T[8] * T[8];
        const float inv = 1.0f / d;
        const float f[3] = {inv, inv, -inv};
        float dT3[3], dL_df[3];
        for (int c = 0; c < 3; ++c) {
            dT[c] += dmx * f[c] * T[6 + c];
            dT[3 + c] += dmy * f[c] * T[6 + c];
            dT3[c] = dmx * f[c] * T[c] + dmy * f[c] * T[3 + c];
            dL_df[c] = dmx * T[c] * T[6 + c] + dmy * T[3 + c] * T[6 + c];
        }
        const float dL_dd = (dL_df[0] * f[0] + dL_df[1] * f[1] + dL_df[2] * f[2]) * (-1.0f / d);
        const float sgn[3] = {1.f, 1.f, -1.f};
        for (int c = 0; c < 3; ++c) dT[6 + c] += dT3[c] + dL_dd * (sgn[c] * T[6 + c] * 2.0f);
        const float Wc = o->focal_x * in->tanfovx, Hc = o->focal_y * in->tanfovy;
        dL_dmeans2D[3 * (size_t)i] = dT[2] * T[8] * Wc;
        dL_dmeans2D[3 * (size_t)i + 1] = dT[5] * T[8] * Hc;
        dL_dmeans2D[3 * (size_t)i + 2] = 0.0f;
    }
    if (dL_dtransMat) for (int k = 0; k < 9; ++k) dL_dtransMat[9 * (size_t)i + k] = dT[k];
    const float* v = in->viewmatrix;
    const float fx = o->focal_x, fy = o->focal_y, cx = fx * in->tanfovx, cy = fy * in->tanfovy;
    float R[3][3];
    {
        const float* q = in->rotations + 4 * (size_t)i;
        const float s = 1.0f / sqrtf(q[3] * q[3] + q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
        const float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
        R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y + w * z); R[0][2] = 2.f * (x * z - w * y);
        R[1][0] = 2.f * (x * y - w * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z + w * x);
        R[2][0] = 2.f * (x * z + w * y); R[2][1] = 2.f * (y * z - w * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
        const float sx = in->scales[2 * (size_t)i], sy = in->scales[2 * (size_t)i + 1];
        const float px = in->means3D[3 * (size_t)i], py = in->means3D[3 * (size_t)i + 1], pz = in->means3D[3 * (size_t)i + 2];
        const float pview[3] = {v[0] * px + v[4] * py + v[8] * pz + v[12], v[1] * px + v[5] * py + v[9] * pz + v[13],
                                v[2] * px + v[6] * py + v[10] * pz + v[14]};
        float dM[3][3], dRS[3][3];
        for (int j = 0; j < 3; ++j) {
            dM[j][0] = fx * dT[j]; dM[j][1] = fy * dT[3 + j]; dM[j][2] = cx * dT[j] + cy * dT[3 + j] + dT[6 + j];
            for (int r = 0; r < 3; ++r) dRS[j][r] = v[4 * r] * dM[j][0] + v[4 * r + 1] * dM[j][1] + v[4 * r + 2] * dM[j][2];
        }
        for (int c = 0; c < 3; ++c) dL_dmeans3D[3 * (size_t)i + c] = dRS[2][c];
        const float dnx = (float)dnrm[3 * (size_t)i], dny = (float)dnrm[3 * (size_t)i + 1], dnz = (float)dnrm[3 * (size_t)i + 2];
        float dtn[3], tn[3];
        for (int r = 0; r < 3; ++r) {
            dtn[r] = v[4 * r] * dnx + v[4 * r + 1] * dny + v[4 * r + 2] * dnz;
            tn[r] = v[r] * R[2][0] + v[4 + r] * R[2][1] + v[8 + r] * R[2][2];
        }
        const float cosv = -(tn[0] * pview[0] + tn[1] * pview[1] + tn[2] * pview[2]);
        const float mult = cosv > 0 ? 1.f : -1.f;
        float vR[3][3];
        for (int r = 0; r < 3; ++r) { vR[0][r] = dRS[0][r] * sx; vR[1][r] = dRS[1][r] * sy; vR[2][r] = dtn[r] * mult; }
        float* dq = dL_drot + 4 * (size_t)i;
        dq[0] = 2.f * (x * (vR[1][2] - vR[2][1]) + y * (vR[2][0] - vR[0][2]) + z * (vR[0][1] - vR[1][0]));
        dq[1] = 2.f * (-2.f * x * (vR[1][1] + vR[2][2]) + y * (vR[0][1] + vR[1][0]) + z * (vR[0][2] + vR[2][0]) + w * (vR[1][2] - vR[2][1]));
        dq[2] = 2.f * (x * (vR[0][1] + vR[1][0]) - 2.f * y * (vR[0][0] + vR[2][2]) + z * (vR[1][2] + vR[2][1]) + w * (vR[2][0] - vR[0][2]));
        dq[3] = 2.f * (x * (vR[0][2] + vR[2][0]) + y * (vR[1][2] + vR[2][1]) - 2.f * z * (vR[0][0] + vR[1][1]) + w * (vR[0][1] - vR[1][0]));
        dL_dscales[2 * (size_t)i] = dRS[0][0] * R[0][0] + dRS[0][1] * R[0][1] + dRS[0][2] * R[0][2];
        dL_dscales[2 * (size_t)i + 1] = dRS[1][0] * R[1][0] + dRS[1][1] * R[1][1] + dRS[1][2] * R[1][2];
    }
    if (in->shs == NULL || in->colors_precomp != NULL) return;
    /* SH backward */
    const int M = in->M, deg = in->D;
    const float* sh = in->shs + (size_t)i * 3 * M;
    float* dsh = dL_dsh + (size_t)i * 3 * M;
    float g[3];
    for (int c = 0; c < 3; ++c) g[c] = o->clamped[3 * (size_t)i + c] ? 0.0f : (float)dcol[3 * (size_t)i + c];
    const float dox = in->means3D[3 * (size_t)i] - in->campos[0], doy = in->means3D[3 * (size_t)i + 1] - in->campos[1],
                doz = in->means3D[3 * (size_t)i + 2] - in->campos[2];
    const float len = sqrtf(dox * dox + doy * doy + doz * doz);
    const float x = dox / len, y = doy / len, z = doz / len;
    float coef[16] = {0};
    float ddx[3] = {0, 0, 0}, ddy[3] = {0, 0, 0}, ddz[3] = {0, 0, 0};
#define SHV(k, c) sh[3 * (k) + (c)]
    coef[0] = SH_C0;
    if (deg > 0) {
        coef[1] = -SH_C1 * y; coef[2] = SH_C1 * z; coef[3] = -SH_C1 * x;
        for (int c = 0; c < 3; ++c) { ddx[c] = -SH_C1 * SHV(3, c); ddy[c] = -SH_C1 * SHV(1, c); ddz[c] = SH_C1 * SHV(2, c); }
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            coef[4] = SH_C2[0] * xy; coef[5] = SH_C2[1] * yz; coef[6] = SH_C2[2] * (2.f * zz - xx - yy);
            coef[7] = SH_C2[3] * xz; coef[8] = SH_C2[4] * (xx - yy);
            for (int c = 0; c < 3; ++c) {
                ddx[c] += SH_C2[0] * y * SHV(4, c) + SH_C2[2] * 2.f * -x * SHV(6, c) + SH_C2[3] * z * SHV(7, c) + SH_C2[4] * 2.f * x * SHV(8, c);
                ddy[c] += SH_C2[0] * x * SHV(4, c) + SH_C2[1] * z * SHV(5, c) + SH_C2[2] * 2.f * -y * SHV(6, c) + SH_C2[4] * 2.f * -y * SHV(8, c);
                ddz[c] += SH_C2[1] * y * SHV(5, c) + SH_C2[2] * 2.f * 2.f * z * SHV(6, c) + SH_C2[3] * x * SHV(7, c);
            }
            if (deg > 2) {
                coef[9] = SH_C3[0] * y * (3.f * xx - yy); coef[10] = SH_C3[1] * xy * z;
                coef[11] = SH_C3[2] * y * (4.f * zz - xx - yy); coef[12] = SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
                coef[13] = SH_C3[4] * x * (4.f * zz - xx - yy); coef[14] = SH_C3[5] * z * (xx - yy);
                coef[15] = SH_C3[6] * x * (xx - 3.f * yy);
                for (int c = 0; c < 3; ++c) {
                    ddx[c] += SH_C3[0] * SHV(9, c) * 3.f * 2.f * xy + SH_C3[1] * SHV(10, c) * yz + SH_C3[2] * SHV(11, c) * -2.f * xy +
                              SH_C3[3] * SHV(12, c) * -3.f * 2.f * xz + SH_C3[4] * SHV(13, c) * (-3.f * xx + 4.f * zz - yy) +
                              SH_C3[5] * SHV(14, c) * 2.f * xz + SH_C3[6] * SHV(15, c) * 3.f * (xx - yy);
                    ddy[c] += SH_C3[0] * SHV(9, c) * 3.f * (xx - yy) + SH_C3[1] * SHV(10, c) * xz +
                              SH_C3[2] * SHV(11, c) * (-3.f * yy + 4.f * zz - xx) + SH_C3[3] * SHV(12, c) * -3.f * 2.f * yz +
                              SH_C3[4] * SHV(13, c) * -2.f * xy + SH_C3[5] * SHV(14, c) * -2.f * yz + SH_C3[6] * SHV(15, c) * -3.f * 2.f * xy;
                    ddz[c] += SH_C3[1] * SHV(10, c) * xy + SH_C3[2] * SHV(11, c) * 4.f * 2.f * yz +
                              SH_C3[3] * SHV(12, c) * 3.f * (2.f * zz - xx - yy) + SH_C3[4] * SHV(13, c) * 4.f * 2.f * xz +
                              SH_C3[5] * SHV(14, c) * (xx - yy);
                }
            }
        }
    }
#undef SHV
    const int ncoef = (deg + 1) * (deg + 1);
    for (int k = 0; k < M && k < ncoef; ++k) for (int c = 0; c < 3; ++c) dsh[3 * k + c] = coef[k] * g[c];
    const float ddir[3] = {ddx[0] * g[0] + ddx[1] * g[1] + ddx[2] * g[2], ddy[0] * g[0] + ddy[1] * g[1] + ddy[2] * g[2],
                           ddz[0] * g[0] + ddz[1] * g[1] + ddz[2] * g[2]};
    const float sum2 = dox * dox + doy * doy + doz * doz;
    const float invs = 1.0f / sqrtf(sum2 * sum2 * sum2);
    dL_dmeans3D[3 * (size_t)i] += ((sum2 - dox * dox) * ddir[0] - doy * dox * ddir[1] - doz * dox * ddir[2]) * invs;
    dL_dmeans3D[3 * (size_t)i + 1] += (-dox * doy * ddir[0] + (sum2 - doy * doy) * ddir[1] - doz * doy * ddir[2]) * invs;
    dL_dmeans3D[3 * (size_t)i + 2] += (-dox * doz * ddir[0] - doy * doz * ddir[1] + (sum2 - doz * doz) * ddir[2]) * invs;
}

/* Rasterizer::backward (rasterizer_impl.cu:346-448).  All outputs must be zero-initialised
 * by the caller, like the reference's torch::zeros (rasterize_points.cu:194-202). */
int oracle_backward(const Oracle* o, const float* dL_dpix, const float* dL_dothers,
                    float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors, float* dL_dopacity,
                    float* dL_dscales, float* dL_drot, float* dL_dtransMat) {
    const int P = o->in.P;
    if (P == 0) return 0;
    double* buf = (double*)calloc((size_t)P * 18, sizeof(double));
    if (!buf) return 1;
    double* dT = buf; double* dm2 = dT + (size_t)P * 9; double* dn = dm2 + (size_t)P * 2;
    double* dop = dn + (size_t)P * 3; double* dc = dop + (size_t)P;
    blend_backward(o, dL_dpix, dL_dothers, dT, dm2, dn, dop, dc);
    for (int i = 0; i < P; ++i) {
        dL_dopacity[i] = (float)dop[i];
        if (dL_dcolors) for (int c = 0; c < 3; ++c) dL_dcolors[3 * (size_t)i + c] = (float)dc[3 * (size_t)i + c];
    }
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; ++i)
        preprocess_backward_one(o, i, dT, dm2, dn, dc, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dscales, dL_drot, dL_dtransMat);
    free(buf);
    return 0;
}

/* accessors for the Python wrapper */
int oracle_ntiles(const Oracle* o) { return o->ntiles; }
uint32_t oracle_num_rendered(const Oracle* o) { return o->num_rendered; }
const int* oracle_radii(const Oracle* o) { return o->radii; }
const float* oracle_depths(const Oracle* o) { return o->depths; }
const float* oracle_transmat(const Oracle* o) { return o->T; }
const float* oracle_center(const Oracle* o) { return o->center; }
const float* oracle_normal(const Oracle* o) { return o->normal; }
const float* oracle_rgb(const Oracle* o) { return o->rgb; }
const uint8_t* oracle_clamped(const Oracle* o) { return o->clamped; }
const uint32_t* oracle_tiles_touched(const Oracle* o) { return o->tiles_touched; }
const uint32_t* oracle_point_list(const Oracle* o) { return o->point_list; }
const uint32_t* oracle_masks(const Oracle* o) { return o->masks; }
const uint32_t* oracle_ranges(const Oracle* o) { return o->ranges; }
const float* oracle_accum(const Oracle* o) { return o->accum; }
const uint32_t* oracle_n_contrib(const Oracle* o) { return o->n_contrib; }
const float* oracle_out_color(const Oracle* o) { return o->out_color; }
const float* oracle_out_others(const Oracle* o) { return o->out_others; }
int oracle_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------------------------------------------------------
 * Float64 replay of the blend under a forward's own decisions, with a running error bound (oracle_replay).
 *
 * Inputs are a forward state from outside -- the per-Gaussian records (T, centre, opacity, normal, colour), the tile
 * lists, each pixel's last and median contributor and the contribution record -- plus the background and upstream
 * gradients.  Which pairs a pixel blended is the record's bit below the pixel's last contributor; which footprint a
 * pair takes (rho3d <= rho2d) is not recorded and is taken from the fp32 sequence of eval_pair (pair_footprints), or
 * from `lowpass` when the caller fixes it.  Pairs whose footprint float64 would choose otherwise are counted, and the
 * Gaussians they touch are flagged: an fp32 kernel may take either branch there.
 *
 * Everything else is recomputed in double from the records (treated as exact): alpha, G, depth, the transmittance,
 * the accumulations and T_final (the images), then the backward of backward.cu:143-449 per pair and its per-Gaussian
 * sums, dT[9], dmean2D[2], dnormal[3], dopacity, dcolor[3].
 *
 * The bound.  Each value v carries e >= |v_fp32 - v|, where v_fp32 is what an fp32 evaluation of the same formula
 * from the same records can return.  With K = 2^-23 (one fp32 ulp relative, twice the unit roundoff of round-to-
 * nearest), first-order running error analysis gives, per operation on inputs (a, ea), (b, eb):
 *   a +- b : ea + eb + K (|a| + |b|)          -- the summands' magnitudes, not the sum's, so that the bound holds for
 *                                                whatever association the kernel uses within a short sum;
 *   a * b  : |a| eb + |b| ea + ea eb + K |ab|
 *   fma    : as a * b + c with one rounding of the result;
 *   a / b  : (ea + |a/b| eb) / (|b| - eb) + 2K |a/b|     -- MUFU.RCP (1 ulp, PTX ISA rcp.approx) and a multiply;
 *   exp(-r/2) : G (expm1(er/2) + 2K + K r/2)           -- 2 ulp (ex2.approx / expf) plus the rounding of the scaled
 *                                                argument, r/2 <= ln 255 for a blended pair.
 * Constants rounded to fp32 carry K/2 relative.  The transmittance the kernel uses at a pair is T_final / prod(1 -
 * alpha_j) over the pairs behind it: its relative bound is T_final's (the forward's own product, bounded as above)
 * plus, per step of the recursion T <- T / (1 - alpha), e(1 - alpha) / (1 - alpha) + 2K, so it grows with the step
 * count.  A per-Gaussian sum of n pair terms x_i, added in any order (red.add), carries sum e_i + (n - 1) K sum |x_i|.
 * Nothing in the bound is fitted to an observed error.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct { double v, e; } B;
#define RK (1.0 / 8388608.0)
static inline B bx(double v) { B r = {v, 0.0}; return r; }
static inline B bc(double v) { B r = {v, 0.5 * RK * fabs(v)}; return r; }       /* constant rounded to fp32 */
static inline B badd(B a, B b) { B r = {a.v + b.v, a.e + b.e + RK * (fabs(a.v) + fabs(b.v))}; return r; }
static inline B bsub(B a, B b) { B r = {a.v - b.v, a.e + b.e + RK * (fabs(a.v) + fabs(b.v))}; return r; }
static inline B bneg(B a) { B r = {-a.v, a.e}; return r; }
static inline B bmul(B a, B b) {
    const double v = a.v * b.v;
    B r = {v, fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e + RK * fabs(v)};
    return r;
}
static inline B bfma(B a, B b, B c) {
    const double v = a.v * b.v + c.v;
    B r = {v, fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e + c.e + RK * fabs(v)};
    return r;
}
static inline B bdiv(B a, B b) {
    const double v = a.v / b.v, d = fabs(b.v) - b.e;
    B r = {v, d > 0.0 ? (a.e + fabs(v) * b.e) / d + 2.0 * RK * fabs(v) : INFINITY};
    return r;
}

typedef struct {
    int P, H, W;
    const double* T;          /* [P,9]: Tu, Tv, Tw */
    const double* center;     /* [P,2] */
    const double* opacity;    /* [P] */
    const double* normal;     /* [P,3] */
    const double* rgb;        /* [P,3] */
    const uint32_t* ranges;   /* [ntiles,2] */
    const uint32_t* point_list;
    const uint32_t* n_contrib;/* [2,H,W] last, median contributor */
    const uint32_t* masks;    /* [8, mask_stride] */
    long long mask_stride;
    const uint8_t* tiles;     /* [ntiles] tiles to replay, or NULL for all */
    const float* bg;          /* [3] */
    const float* dL_dpix;     /* [3,H,W] */
    const float* dL_dothers;  /* [8,H,W] */
    uint8_t* lowpass;         /* NULL, or [num_rendered, 256] footprint choice per (list position, tile pixel) */
    int fix_lowpass;          /* 1: read `lowpass`; 0: write it (when given) */
} ReplayIn;

#define RG 18   /* per-Gaussian partials: dT[9], dmean2D[2], dnormal[3], dopacity, dcolor[3] */

typedef struct {
    double* img;      /* [14,H,W] colour[3], others[8], accum[3] (T_final, dist1, dist2); zeroed by the caller */
    double* img_e;    /* [14,H,W] their bounds */
    double* g;        /* [P,RG] zeroed by the caller */
    double* g_e;      /* [P,RG] */
    int64_t* npairs;  /* [P] blended pairs per Gaussian; zeroed */
    int64_t* nlow;    /* [P] of which low-pass; zeroed */
    uint8_t* band;    /* [P] 1 = touched by a pair whose footprint float64 chooses otherwise; zeroed */
    int64_t counts[4];/* pairs, low-pass pairs, band pairs, pixels replayed */
} ReplayOut;

typedef struct {
    B kx, ky, kz, lx, ly, lz, px, py, pz, sx, sy, depth, G, alpha;
    double dx, dy;
    int lowpass, band;
} RPair;

static void replay_pair(const ReplayIn* in, uint32_t g, float pixx, float pixy, int lp_fixed, RPair* r) {
    const double* T = in->T + 9 * (size_t)g;
    const B T0 = bx(T[0]), T1 = bx(T[1]), T2 = bx(T[2]), T3 = bx(T[3]), T4 = bx(T[4]), T5 = bx(T[5]);
    const B T6 = bx(T[6]), T7 = bx(T[7]), T8 = bx(T[8]);
    const B X = bx(pixx), Y = bx(pixy);
    r->kx = bfma(X, T6, bneg(T0)); r->ky = bfma(X, T7, bneg(T1)); r->kz = bfma(X, T8, bneg(T2));
    r->lx = bfma(Y, T6, bneg(T3)); r->ly = bfma(Y, T7, bneg(T4)); r->lz = bfma(Y, T8, bneg(T5));
    r->pz = bfma(r->kx, r->ly, bneg(bmul(r->ky, r->lx)));
    r->px = bfma(r->ky, r->lz, bneg(bmul(r->kz, r->ly)));
    r->py = bfma(r->kz, r->lx, bneg(bmul(r->kx, r->lz)));
    r->sx = bdiv(r->px, r->pz); r->sy = bdiv(r->py, r->pz);
    const B rho3d = bfma(r->sx, r->sx, bmul(r->sy, r->sy));
    r->dx = in->center[2 * (size_t)g] - pixx; r->dy = in->center[2 * (size_t)g + 1] - pixy;
    const B dx = {r->dx, RK * fabs(r->dx)}, dy = {r->dy, RK * fabs(r->dy)};
    const B rho2d = bmul(bx(2.0), bfma(dx, dx, bmul(dy, dy)));
    int lp;
    if (lp_fixed >= 0) {
        lp = lp_fixed;
    } else {
        float Tf[9], cf[2];
        for (int k = 0; k < 9; ++k) Tf[k] = (float)T[k];
        cf[0] = (float)in->center[2 * (size_t)g]; cf[1] = (float)in->center[2 * (size_t)g + 1];
        Pair e;
        lp = pair_footprints(Tf, cf, pixx, pixy, &e) ? !(e.rho3d <= e.rho2d) : 1;
    }
    r->lowpass = lp;
    r->band = lp != !(rho3d.v <= rho2d.v);
    const B rho = lp ? rho2d : rho3d;
    r->depth = lp ? T8 : badd(T8, bfma(T6, r->sx, bmul(T7, r->sy)));
    const double G = exp(-0.5 * rho.v);
    r->G.v = G;
    r->G.e = G * (expm1(0.5 * rho.e) + 2.0 * RK + RK * 0.5 * fabs(rho.v));
    B a = bmul(bx(in->opacity[g]), r->G);
    if (a.v > 0.99) { a.e = a.v - a.e > 0.99 ? 0.0 : a.e; a.v = 0.99; }   /* min(0.99, .) */
    r->alpha = a;
}

static inline void acc_g(double* g, double* ge, double* gs, size_t i, int k, B x) {
    atomic_add_d(&g[i * RG + k], x.v);
    atomic_add_d(&ge[i * RG + k], x.e);
    atomic_add_d(&gs[i * RG + k], fabs(x.v));
}

int oracle_replay(const ReplayIn* in, ReplayOut* out) {
    const int H = in->H, W = in->W, P = in->P;
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE, ntiles = gx * gy;
    const size_t npix = (size_t)H * W;
    double* gs = (double*)calloc((size_t)(P > 0 ? P : 1) * RG, sizeof(double));   /* sums of |terms| */
    if (!gs) return 1;
    int64_t c_pairs = 0, c_low = 0, c_band = 0, c_pix = 0;
    const double bgd[3] = {in->bg[0], in->bg[1], in->bg[2]};
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : c_pairs, c_low, c_band, c_pix)
    for (int tile = 0; tile < ntiles; ++tile) {
        if (in->tiles && !in->tiles[tile]) continue;
        const int ty = tile / gx, tx = tile % gx;
        const uint32_t r0 = in->ranges[2 * tile];
        for (int ly = 0; ly < TILE; ++ly) for (int lx = 0; lx < TILE; ++lx) {
            const int x = tx * TILE + lx, y = ty * TILE + ly;
            if (x >= W || y >= H) continue;
            const size_t pix = (size_t)y * W + x;
            const float pixx = (float)x + 0.5f, pixy = (float)y + 0.5f;
            const int last = (int)in->n_contrib[pix], median = (int)in->n_contrib[pix + npix];
            const uint32_t* mrow = in->masks + (size_t)((ly >> 2) * 2 + (lx >> 3)) * in->mask_stride + r0;
            const uint32_t bit = 1u << ((ly & 3) * 8 + (lx & 7));
            const int tp = ly * TILE + lx;
            ++c_pix;
            /* ---- forward under the recorded decisions */
            B Tr = bx(1.0), C[3] = {bx(0), bx(0), bx(0)}, N[3] = {bx(0), bx(0), bx(0)}, D = bx(0);
            B dist1 = bx(0), dist2 = bx(0), distortion = bx(0), med_d = bx(0), med_w = bx(0);
            for (int pos = 0; pos < last; ++pos) {
                if (!(mrow[pos] & bit)) continue;
                const uint32_t g = in->point_list[r0 + pos];
                RPair e;
                uint8_t* lpp = in->lowpass ? in->lowpass + (size_t)(r0 + pos) * 256 + tp : NULL;
                replay_pair(in, g, pixx, pixy, (lpp && in->fix_lowpass) ? *lpp : -1, &e);
                if (lpp && !in->fix_lowpass) *lpp = (uint8_t)e.lowpass;
                const B al = e.alpha, w = bmul(al, Tr);
                const B A = bsub(bx(1.0), Tr);
                const double m_v = (100.0 * e.depth.v - 20.0) / (99.8 * e.depth.v);
                const B m = {m_v, 0.2004008 / (e.depth.v * e.depth.v) * e.depth.e + RK * (1.0 + fabs(m_v))};
                const B mm = bmul(m, m);
                const B err = bfma(bneg(dist1), badd(m, m), bfma(A, mm, dist2));
                distortion = bfma(w, err, distortion);
                if (pos == median - 1) { med_d = e.depth; med_w = w; }
                for (int c = 0; c < 3; ++c) N[c] = bfma(w, bx(in->normal[3 * (size_t)g + c]), N[c]);
                D = bfma(w, e.depth, D);
                dist1 = bfma(w, m, dist1);
                dist2 = bfma(w, mm, dist2);
                for (int c = 0; c < 3; ++c) C[c] = bfma(w, bx(in->rgb[3 * (size_t)g + c]), C[c]);
                Tr = bmul(Tr, bsub(bx(1.0), al));
                ++c_pairs; c_low += e.lowpass; c_band += e.band;
                if (e.band) out->band[g] = 1;
            }
            const B Tf = Tr;
            const B img[14] = {bfma(bx(bgd[0]), Tf, C[0]), bfma(bx(bgd[1]), Tf, C[1]), bfma(bx(bgd[2]), Tf, C[2]),
                               D, bsub(bx(1.0), Tf), N[0], N[1], N[2], med_d, distortion, med_w, Tf, dist1, dist2};
            for (int k = 0; k < 14; ++k) { out->img[k * npix + pix] = img[k].v; out->img_e[k * npix + pix] = img[k].e; }

            /* ---- backward, back to front (backward.cu:321-446) */
            float up[11];
            for (int c = 0; c < 3; ++c) up[c] = in->dL_dpix[pix + c * npix];
            for (int c = 0; c < 8; ++c) up[3 + c] = in->dL_dothers[pix + c * npix];
            int nz = 0;
            for (int c = 0; c < 11; ++c) nz |= up[c] != 0.0f;
            if (!nz) continue;
            const B dpix[3] = {bx(up[0]), bx(up[1]), bx(up[2])};
            const B dL_ddepth = bx(up[3]), dL_daccum = bx(up[4]), dn[3] = {bx(up[5]), bx(up[6]), bx(up[7])};
            const B dL_dmed = bx(up[8]), dL_dreg = bx(up[9]), dL_dmaxw = bx(up[10]);
            const B final_A = bsub(bx(1.0), Tf);
            const B bg_dot = badd(badd(bmul(bx(bgd[0]), dpix[0]), bmul(bx(bgd[1]), dpix[1])), bmul(bx(bgd[2]), dpix[2]));
            const B nTf_bg = bneg(bmul(Tf, bg_dot));
            const B A_r = bmul(final_A, dL_dreg), nD_r = bmul(bmul(bx(-2.0), dist1), dL_dreg), D2_r = bmul(dist2, dL_dreg);
            const B c2 = bc(20.0 / 99.8);
            /* the eight recursions of accum_rec: colour, depth, normal, alpha; and their upstream gradients */
            B acc[8] = {bx(0), bx(0), bx(0), bx(0), bx(0), bx(0), bx(0), bx(0)};
            const B dch[8] = {dpix[0], dpix[1], dpix[2], dL_ddepth, dn[0], dn[1], dn[2], dL_daccum};
            B last_dL_dT = bx(0);
            double Tv = Tf.v, relT = Tf.v > 0.0 ? Tf.e / Tf.v : INFINITY;
            for (int pos = last - 1; pos >= 0; --pos) {
                if (!(mrow[pos] & bit)) continue;
                const uint32_t g = in->point_list[r0 + pos];
                RPair e;
                const uint8_t* lpp = in->lowpass ? in->lowpass + (size_t)(r0 + pos) * 256 + tp : NULL;
                replay_pair(in, g, pixx, pixy, lpp ? *lpp : -1, &e);
                const B al = e.alpha, om = bsub(bx(1.0), al);
                Tv = Tv / om.v;
                relT += om.e / om.v + 2.0 * RK;
                const B T = {Tv, Tv * relT};
                const B w = bmul(al, T);
                const B cur[8] = {bx(in->rgb[3 * (size_t)g]), bx(in->rgb[3 * (size_t)g + 1]), bx(in->rgb[3 * (size_t)g + 2]),
                                  e.depth, bx(in->normal[3 * (size_t)g]), bx(in->normal[3 * (size_t)g + 1]),
                                  bx(in->normal[3 * (size_t)g + 2]), bx(1.0)};
                B dsum = bx(0);
                for (int c = 0; c < 8; ++c) {
                    const B d = bsub(cur[c], acc[c]);
                    dsum = bfma(d, dch[c], dsum);
                    acc[c] = bfma(d, al, acc[c]);
                }
                B dL_dz = bmul(w, dL_ddepth);
                const B rcd = bdiv(bx(1.0), e.depth);
                const B m = bsub(bc(100.0 / 99.8), bmul(c2, rcd));
                B dL_dweight = bfma(m, bfma(m, A_r, nD_r), D2_r);
                if (pos == median - 1) { dL_dz = badd(dL_dz, dL_dmed); dL_dweight = badd(dL_dweight, dL_dmaxw); }
                const B ddw = bsub(dL_dweight, last_dL_dT);
                B dL_dalpha = badd(dsum, ddw);
                last_dL_dT = bfma(al, ddw, last_dL_dT);
                /* dL_dmd * dm/dd = 2 w (m A - D) dL_dreg * c2 / d^2 */
                dL_dz = bfma(bmul(w, bfma(m, bmul(bmul(bx(2.0), c2), A_r), bmul(c2, nD_r))), bmul(rcd, rcd), dL_dz);
                dL_dalpha = bmul(dL_dalpha, T);
                dL_dalpha = badd(dL_dalpha, bdiv(nTf_bg, om));
                const B GdA = bmul(e.G, dL_dalpha);
                const B opac = bx(in->opacity[g]);
                for (int c = 0; c < 3; ++c) {
                    acc_g(out->g, out->g_e, gs, g, 15 + c, bmul(w, dpix[c]));
                    acc_g(out->g, out->g_e, gs, g, 11 + c, bmul(w, dn[c]));
                }
                acc_g(out->g, out->g_e, gs, g, 14, GdA);
                if (!e.lowpass) {
                    /* vjp through s = p.xy / p.z, p = k x l (backward.cu:405-435) */
                    const B nOG = bneg(bmul(opac, GdA));
                    const B dsx = bfma(e.sx, nOG, bmul(bx(in->T[9 * (size_t)g + 6]), dL_dz));
                    const B dsy = bfma(e.sy, nOG, bmul(bx(in->T[9 * (size_t)g + 7]), dL_dz));
                    const B dp0 = bdiv(dsx, e.pz), dp1 = bdiv(dsy, e.pz);
                    const B dp2 = bneg(badd(bmul(dp0, e.sx), bmul(dp1, e.sy)));
                    const B dk[3] = {bsub(bmul(e.ly, dp2), bmul(e.lz, dp1)), bsub(bmul(e.lz, dp0), bmul(e.lx, dp2)),
                                     bsub(bmul(e.lx, dp1), bmul(e.ly, dp0))};
                    const B dl[3] = {bsub(bmul(dp1, e.kz), bmul(dp2, e.ky)), bsub(bmul(dp2, e.kx), bmul(dp0, e.kz)),
                                     bsub(bmul(dp0, e.ky), bmul(dp1, e.kx))};
                    const B dzw[3] = {e.sx, e.sy, bx(1.0)};
                    for (int c = 0; c < 3; ++c) {
                        acc_g(out->g, out->g_e, gs, g, c, bneg(dk[c]));
                        acc_g(out->g, out->g_e, gs, g, 3 + c, bneg(dl[c]));
                        acc_g(out->g, out->g_e, gs, g, 6 + c,
                              bfma(bx(pixx), dk[c], bfma(bx(pixy), dl[c], bmul(dL_dz, dzw[c]))));
                    }
                } else {
                    /* low-pass branch (backward.cu:436-443), FilterInvSquare = 2 */
                    const B k = bmul(bx(-2.0), bmul(opac, GdA));
                    acc_g(out->g, out->g_e, gs, g, 9, bmul(k, (B){e.dx, RK * fabs(e.dx)}));
                    acc_g(out->g, out->g_e, gs, g, 10, bmul(k, (B){e.dy, RK * fabs(e.dy)}));
                    acc_g(out->g, out->g_e, gs, g, 8, dL_dz);
                }
#pragma omp atomic
                out->npairs[g] += 1;
                if (e.lowpass) {
#pragma omp atomic
                    out->nlow[g] += 1;
                }
            }
        }
    }
    /* summation bound of the per-Gaussian sums, in any order */
    for (int i = 0; i < P; ++i) {
        const double n1 = out->npairs[i] > 1 ? (double)(out->npairs[i] - 1) : 0.0;
        for (int k = 0; k < RG; ++k) out->g_e[(size_t)i * RG + k] += n1 * RK * gs[(size_t)i * RG + k];
    }
    free(gs);
    out->counts[0] = c_pairs; out->counts[1] = c_low; out->counts[2] = c_band; out->counts[3] = c_pix;
    return 0;
}
