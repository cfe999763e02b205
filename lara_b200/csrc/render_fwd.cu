// render_fwd.cu -- per-tile front-to-back alpha compositing (K6).
// Replaces reference forward.cu:265-463 (renderCUDA forward).
//
// One CTA (SRF_CTA_WARPS = 8 warps) per 16x16 tile, one thread per pixel (each warp owns an
// 8x4 pixel block).  The tile's depth-sorted Gaussian list is consumed in rounds of SRF_BATCH
// = 256: every thread gathers one 96 B GeomRecord with six 128-bit loads, stages what the blend
// reads in shared memory, so the inner loop never touches global memory -- including the colour,
// which the reference fetches from global memory per contributing pixel -- and culls the splat
// against the tile's eight 8x4 blocks once (one byte per batch slot).  Per round each warp then
// builds per-pixel hit masks (the splat's conservative alpha >= 1/255 octagon rasterised over the
// warp's block, transposed across the warp) and every lane walks its own hits in list order,
// reading the records at per-lane indices (phases A / B below).  Arithmetic and predicates follow
// the reference exactly (see eval_pair()).
// Every warp also records, per list position, which pixels of its block the splat was blended into (one u32
// per (position, 8x4 block), RenderFwdArgs::masks): the blend backward replays that record instead of culling,
// masking and re-testing the pairs itself.
// The forward-only instantiation (kRecord = false, for renders no gradient flows through) keeps the hit masks, the walk,
// eval_pair, the saturation test and the output stores, and drops everything that serves only the backward: the record
// (s_out, its clearing, the transposes back and the stores, the lanes' blended-bit write-backs into s_mask) and the
// accum / n_contrib image state.  Its outputs are bit-identical to the training instantiation's.
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

// The staged record in shared memory, as phase B reads it: four float4 planes q0, q1, q2 and (n.x, n.y, n.z, r), the
// colour's (g, b) as one float2 plane, and the cull octagon q5, which only the pixel masks read.  A contributing trip reads
// normal and colour with one 16-byte and one 8-byte load; the view-space depth q3.w and the clamp bits q4.w, which the
// blend never reads, are not staged.  Byte offsets of the planes:
constexpr uint32_t kFwdQ3 = 16u * 3 * SRF_BATCH;          // (n.x, n.y, n.z, r)
constexpr uint32_t kFwdGB = 16u * 4 * SRF_BATCH;          // (g, b)
constexpr uint32_t kFwdOct = kFwdGB + 8u * SRF_BATCH;     // q5
constexpr uint32_t kFwdRecBytes = kFwdOct + 16u * SRF_BATCH;

template <bool kRecord>
__global__ void __launch_bounds__(SRF_CTA_THREADS, 1024 / SRF_CTA_THREADS) render_fwd_kernel(RenderFwdArgs a) {
    __shared__ __align__(16) uint8_t s_rec[kFwdRecBytes];
    __shared__ uint8_t s_blk[SRF_BATCH];                               // [batch slot]: bit b = may touch the tile's block b
    __shared__ uint32_t s_mask[SRF_CTA_WARPS][SRF_BATCH_CHUNKS][32];   // [warp][group of 32 hits][lane]: per-pixel hit words
    __shared__ uint8_t s_list[SRF_CTA_WARPS][SRF_BATCH];               // [warp]: batch slots of the splats that can touch the warp's block
    __shared__ __align__(16) uint32_t s_out[SRF_CTA_WARPS][SRF_BATCH];  // [warp][batch slot]: contribution masks of the batch
                                                                        // (not referenced, so not allocated, without kRecord)
    float4* const s_q = reinterpret_cast<float4*>(s_rec);               // s_q[k * SRF_BATCH + slot]: float4 plane k
    const float4* const s_q5 = reinterpret_cast<const float4*>(s_rec + kFwdOct);

    const int tid = threadIdx.x;
    {   // view of this CTA: per-view workspaces of identical layout, images stacked [V,C,H,W]
        const int view = blockIdx.y;
        const size_t npix_v = (size_t)a.W * a.H;
        a.ranges = view_ptr(a.ranges, view, a.tile_stride);
        a.tile_order = view_ptr(a.tile_order, view, a.tile_stride);
        a.point_list = view_ptr(a.point_list, view, a.plist_stride);
        a.masks = view_ptr(a.masks, view, a.plist_stride);
        a.rec = view_ptr(a.rec, view, a.geom_stride);
        a.bg += (size_t)view * a.cam_stride;
        a.accum = view_ptr(a.accum, view, a.image_stride);
        a.n_contrib = view_ptr(a.n_contrib, view, a.image_stride);
        a.out_color += (size_t)view * 3 * npix_v;
        a.out_others += (size_t)view * 8 * npix_v;
    }
    const int tile = (int)a.tile_order[blockIdx.x / SRF_CTAS_PER_TILE];
    const int gw = (int)(blockIdx.x % SRF_CTAS_PER_TILE) * SRF_CTA_WARPS + (tid >> 5);   // which of the tile's eight 8x4 blocks
    const int tyi = tile / a.gx, txi = tile - tyi * a.gx;
    int lx, ly;
    tile_pixel(gw * 32 + (tid & 31), lx, ly);
    const int pxi = txi * SRF_TILE + lx, pyi = tyi * SRF_TILE + ly;
    const bool inside = pxi < a.W && pyi < a.H;
    const float pixx = (float)pxi + 0.5f, pixy = (float)pyi + 0.5f;
    // pixel-centre rectangle of this warp's 8x4 block, for the pixel masks
    const int lane = tid & 31, wid = tid >> 5;
    const WarpRect wrect = make_warp_rect(txi, tyi, gw);

    uint2 range = a.ranges[tile];
    if (range.y > a.capacity) range.y = range.x;  // overflowed optimistic capacity: host re-runs
    const int n = (int)(range.y - range.x);
    const int rounds = (n + SRF_BATCH - 1) / SRF_BATCH;

    bool done = !inside;
    float T = 1.0f;
    uint32_t last_contributor = 0;
    // accumulators, two per f32x2 pair: (C0,C1) (C2,distortion) (N0,N1) (N2,D) (dist1,dist2)
    f32x2 C01 = zero2(), C2r = zero2(), N01 = zero2(), N2D = zero2(), d12 = zero2();
    float median_depth = 0.f, median_weight = 0.f;
    // 1-based list position of the median contributor, 0 = none.  (The reference keeps a float
    // initialised to -1 and converts it to u32 at the end -- 0 after saturation; for tiles with an
    // empty list its compiled code leaves the value uninitialised.)
    uint32_t median_contributor = 0;

    // phase B addresses its shared arrays explicitly (smem_addr): the staged records, the warp's hit list and the lane's
    // hit words
    uint32_t sa_rec = smem_addr(s_rec), sa_list = smem_addr(&s_list[wid][0]), sa_mask = smem_addr(&s_mask[wid][0][lane]);
    asm volatile("" : "+r"(sa_rec), "+r"(sa_list), "+r"(sa_mask));   // opaque: kept in registers, not rebuilt at every use
    // ptxas still rematerialises the record base (S2R SR_CgaCtaId + LEA) at both of its uses in the pair loop; a shuffled
    // copy is a value it cannot recompute
    sa_rec = __shfl_sync(0xffffffffu, sa_rec, 0);

    int todo = n;
    for (int b = 0; b < rounds; ++b, todo -= SRF_BATCH) {
        // whole tile saturated -> stop (reference forward.cu:334-336)
        if (__syncthreads_count(done) == SRF_CTA_THREADS) break;
        // ---- staging and the cull: the thread of batch slot tid stages its splat and tests the splat's conservative
        // alpha >= 1/255 octagon against all eight 8x4 blocks of the tile (octagon_block_bits: bit b is exactly
        // octagon_hits against block b), so each staged splat is culled once for the whole tile.  Slots past the list's
        // end get no bits.
        const int progress = b * SRF_BATCH + tid;
        uint32_t blk = 0;
        if (progress < n) {
            const uint32_t id = __ldg(a.point_list + range.x + progress);
            const float4* r = a.rec + (size_t)id * SRF_REC_QUADS;
            const float4 q2 = ldg4(r + 2), q3 = ldg4(r + 3), q4 = ldg4(r + 4), q5 = ldg4(r + 5);
            s_q[0 * SRF_BATCH + tid] = ldg4(r + 0);
            s_q[1 * SRF_BATCH + tid] = ldg4(r + 1);
            s_q[2 * SRF_BATCH + tid] = q2;
            s_q[3 * SRF_BATCH + tid] = make_float4(q3.x, q3.y, q3.z, q4.x);
            reinterpret_cast<float2*>(s_rec + kFwdGB)[tid] = make_float2(q4.y, q4.z);
            reinterpret_cast<float4*>(s_rec + kFwdOct)[tid] = q5;
            // the tile's block bounds are rebuilt here per batch: hoisted out of the batch loop, their 44 floats
            // do not fit in the registers
            int tx = txi, ty = tyi;
            asm volatile("" : "+r"(tx), "+r"(ty));
            blk = octagon_block_bits(q2, q5, tx, ty);
        }
        s_blk[tid] = (uint8_t)blk;
        __syncthreads();
        const int cnt = min(SRF_BATCH, todo);
        // warp-uniform skip: a fully saturated warp only helps with staging
        if (__all_sync(0xffffffffu, done)) continue;
        // ---- phase A: per-pixel hit masks.  The staged splats whose octagon can touch this warp's 8x4 block at all
        // (~1 in 5: bit gw of their block byte) are compacted into a list, in list order.  Then, 32 hits at a time, lane
        // l rasterises the octagon of hit g*32+l over the block into a 32-bit mask (bit = lane that owns the pixel) and a
        // 32x32 bit transpose over the warp hands every lane the word "which of these 32 splats can touch MY pixel".  A
        // splat outside a pixel's word cannot reach alpha >= 1/255 there, so skipping it changes no result.
        static_assert(SRF_BATCH == 256, "s_out is cleared with two 16-byte stores per lane");
        if constexpr (kRecord) {
            reinterpret_cast<uint4*>(s_out[wid])[lane] = make_uint4(0u, 0u, 0u, 0u);
            reinterpret_cast<uint4*>(s_out[wid])[lane + 32] = make_uint4(0u, 0u, 0u, 0u);
        }
        int nh = 0;
        for (int c0 = 0; c0 < cnt; c0 += 32) {
            const int jt = c0 + lane;
            const bool hit = (s_blk[jt] >> gw) & 1u;   // 0 for slots at or past cnt
            const unsigned hits = __ballot_sync(0xffffffffu, hit);
            if (hit) s_list[wid][nh + __popc(hits & ((1u << lane) - 1u))] = (uint8_t)jt;
            nh += __popc(hits);
        }
        __syncwarp();
        const int nchunks = (nh + 31) >> 5;
        for (int c = 0; c < nchunks; ++c) {
            const int h = (c << 5) + lane;
            uint32_t m = 0;
            if (h < nh) {
                const int jt = s_list[wid][h];
                m = octagon_pixel_mask(s_q[2 * SRF_BATCH + jt], s_q5[jt], wrect);
            }
            s_mask[wid][c][lane] = transpose32(m, lane);
        }
        __syncwarp();

        // ---- phase B: every lane walks its own hits in list order and leaves the loop when it has none left; the warp
        // reconverges once, after the loop.  The lane's hit word is bit-reversed: hit i of the chunk is bit 31 - i, the
        // next one is the highest set bit p (hit 31 - p), and w & bits_below(p) drops it.
        // Each lane also records which of its hits it blended: cw collects the (bit-reversed) bits of chunk c and replaces
        // the lane's (already read) hit word s_mask[wid][c][lane], in list order again, when the lane leaves the chunk.
        const uint32_t cbase = (uint32_t)(b * SRF_BATCH + 1);   // contributor = cbase + batch slot (1-based list position)
        int c = 0;
        uint32_t w = 0, cw = 0;
        if (done) {
            if constexpr (kRecord)
                for (int k = 0; k < nchunks; ++k) sts_u32(sa_mask + 128u * k, 0u);
            c = nchunks;
        } else if (nchunks > 0) {
            w = __brev(lds_u32(sa_mask));
        }
        uint32_t sa_lc = sa_list + 31u;   // hit 31 - p of chunk c is list entry sa_lc - p
        for (;;) {
            while (w == 0 && c < nchunks - 1) {
                if constexpr (kRecord) { sts_u32(sa_mask + 128u * c, __brev(cw)); cw = 0; }
                ++c; sa_lc += 32u; w = __brev(lds_u32(sa_mask + 128u * c));
            }
            if (w == 0) break;
            const int p = 31 - __clz(w);
            w &= bits_below(p);
            const uint32_t j = lds_u8(sa_lc - (uint32_t)p);
            const uint32_t sa_j = sa_rec + 16u * j;
            const float4 q0 = lds_f4(sa_j), q1 = lds_f4(sa_j + 16u * SRF_BATCH), q2 = lds_f4(sa_j + 32u * SRF_BATCH);
            const float4 q3 = lds_f4(sa_j + kFwdQ3);
            const float2 gb = lds_f2(sa_rec + kFwdGB + 8u * j);
            PairEval e;
            eval_pair(q0, q1, q2, pixx, pixy, e);
            if (!e.valid) continue;
            const float alpha = e.alpha;
            const float test_T = fmul_(T, fadd_(1.0f, -alpha));
            if (!(test_T >= 0.0001f)) {
                done = true;
                if constexpr (kRecord) {
                    sts_u32(sa_mask + 128u * c, __brev(cw));
                    for (int k = c + 1; k < nchunks; ++k) sts_u32(sa_mask + 128u * k, 0u);
                }
                c = nchunks;
                break;
            }
            if constexpr (kRecord) cw |= 1u << p;
            const float depth = e.depth;
            const float A = fadd_(1.0f, -T);
            const float m = mapped_depth_fast(depth);
            const float mm = fmul_(m, m);
            const float2 d12_ = up2(d12);
            const float err = fma_(-d12_.x, fadd_(m, m), fma_(A, mm, d12_.y));
            if (T > 0.5f) {
                median_depth = depth;
                median_weight = fmul_(T, alpha);
                median_contributor = cbase + j;
            }
            // every channel: acc = fma(T, channel * alpha, acc) -- the reference's rounding sequence,
            // two channels per mul2 / fma2 pair
            const f32x2 a2 = bc2(alpha), T2 = bc2(T);
            fma2_acc(C01, T2, mul2(pk2(q3.w, gb.x), a2));
            fma2_acc(C2r, T2, mul2(pk2(gb.y, err), a2));
            fma2_acc(N01, T2, mul2(pk2(q3.x, q3.y), a2));
            fma2_acc(N2D, T2, mul2(pk2(q3.z, depth), a2));
            fma2_acc(d12, T2, mul2(pk2(m, mm), a2));
            T = test_T;
            last_contributor = cbase + j;
        }
        // without the record, the next batch's __syncthreads_count orders the reuse of the warp's shared arrays
        if constexpr (kRecord) {
            if (c < nchunks) sts_u32(sa_mask + 128u * c, __brev(cw));
            __syncwarp();

            // ---- contribution record of the batch: transposed back, lane l holds the pixel mask of hit 32 k + l, which
            // goes to its batch slot (the slots the cull dropped stay 0); then 32 consecutive list positions per store
            for (int k = 0; k < nchunks; ++k) {
                const uint32_t m = transpose32(s_mask[wid][k][lane], lane);
                if ((k << 5) + lane < nh) s_out[wid][s_list[wid][(k << 5) + lane]] = m;
            }
            // a warp that saturated in this batch stores only the positions before its block's deepest contributor
            int lim = cnt;
            if (__all_sync(0xffffffffu, done)) lim = min(cnt, (int)__reduce_max_sync(0xffffffffu, last_contributor) - b * SRF_BATCH);
            __syncwarp();
            uint32_t* dst = a.masks + (size_t)gw * a.capacity + range.x + b * SRF_BATCH;
            for (int jt = lane; jt < lim; jt += 32) dst[jt] = s_out[wid][jt];
        }
    }

    const float2 C01_ = up2(C01), C2r_ = up2(C2r), N01_ = up2(N01), N2D_ = up2(N2D), d12_f = up2(d12);
    const float C0 = C01_.x, C1 = C01_.y, C2 = C2r_.x, distortion = C2r_.y;
    const float N0 = N01_.x, N1 = N01_.y, N2 = N2D_.x, D = N2D_.y, dist1 = d12_f.x, dist2 = d12_f.y;
    if (inside) {
        const size_t npix = (size_t)a.W * a.H;
        const size_t pix = (size_t)pyi * a.W + pxi;
        if constexpr (kRecord) {
            a.accum[pix] = T;
            a.accum[pix + npix] = dist1;
            a.accum[pix + 2 * npix] = dist2;
            a.n_contrib[pix] = last_contributor;
            a.n_contrib[pix + npix] = median_contributor;
        }
        a.out_color[pix] = fma_(__ldg(a.bg + 0), T, C0);
        a.out_color[pix + npix] = fma_(__ldg(a.bg + 1), T, C1);
        a.out_color[pix + 2 * npix] = fma_(__ldg(a.bg + 2), T, C2);
        a.out_others[pix] = D;
        a.out_others[pix + npix] = fadd_(1.0f, -T);
        a.out_others[pix + 2 * npix] = N0;
        a.out_others[pix + 3 * npix] = N1;
        a.out_others[pix + 4 * npix] = N2;
        a.out_others[pix + 5 * npix] = median_depth;
        a.out_others[pix + 6 * npix] = distortion;
        a.out_others[pix + 7 * npix] = median_weight;
    }
}

cudaError_t launch_render_fwd(const RenderFwdArgs& a, bool record, cudaStream_t stream) {
    const int ntiles = a.gx * a.gy;
    if (ntiles <= 0 || a.nviews <= 0) return cudaSuccess;
    prof_start(K_RENDER_FWD, stream);
    const dim3 grid(ntiles * SRF_CTAS_PER_TILE, a.nviews);
    if (record)
        render_fwd_kernel<true><<<grid, SRF_CTA_THREADS, 0, stream>>>(a);
    else
        render_fwd_kernel<false><<<grid, SRF_CTA_THREADS, 0, stream>>>(a);
    prof_stop(K_RENDER_FWD, stream);
    return cudaGetLastError();
}

}  // namespace srf
