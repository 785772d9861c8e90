// gsr_features.cu — per-gaussian feature channels blended with the colour's weights (DESIGN.md 3.17), forward and
// backward, one CTA per 16x16 tile and chunk of FCH channels (grid z).
//
// The kernels walk the tile's sorted pair list with the machinery of the colour renderers (gsr_tile_walk.cuh): the
// same 128-thread CTA with two pixels per lane, the same stage ring filled by cp.async on the stage mbarrier (each
// record's FCH feature floats ride along as one more 16-byte copy), the same warp-granular stage recycling and the
// same per-lane-group lists.  They do not change the colour kernels: those keep their code and SASS.
//
// Forward: every rounded operation that decides a blend weight is the one k_render_fwd issues (fwd_walk in
// gsr_render.cu, op for op), and the pixels it flags for the exact recomputation are flagged here by the same tests,
// so w_i is the colour's float, bit for bit.  The forward always rebuilds the candidate lists from the footprints:
// the contribution masks name the records that contributed, but the exact-division range check must also see the
// records that did not (a flag raised by one of them sends the pixel to the exact replay in the colour forward).
//
// Backward: the recurrence of k_render_bwd (back to front from n_per_pixel / w_per_pixel, r = 1/(1-alpha), the
// 0.9999 clamp, the chunk-local weight index), with the colour replaced by FCH feature accumulators and no background.
// Per (gaussian, tile) ten moments are reduced over the lane group and the stage accumulator: the FCH feature
// gradients and the feature loss's part of the six geometry moments, which are linear in d_alpha and are finished and
// added into the interleaved gradient rows exactly as the colour backward finishes its own.
#include "gsr_tile_walk.cuh"

#include "../../include/gsr_features.h"

namespace gsr {

constexpr int FCH = 4;        // feature channels per CTA: one 16-byte copy per record, one v4 reduction per flush
constexpr int NGF = FCH + 6;  // backward moments per record: FCH feature gradients, g*d_alpha, hu, hv, hu*du, hu*dv, hv*dv
static_assert(GROUPS == 4, "the feature backward reduces its moments over quarter-warp lane groups");

#ifndef GSR_FEAT_FWD_MINB
#define GSR_FEAT_FWD_MINB 8
#endif
#ifndef GSR_FEAT_BWD_MINB
#define GSR_FEAT_BWD_MINB 6
#endif

// whole warp: gather_batch plus the chunk's FCH floats of every record (fsrc: the chunk's first column)
__device__ __forceinline__ void gather_batch_features(const RecSource& src, const float* __restrict__ fsrc,
                                                      int stride, int p0, int cnt, float* __restrict__ stage,
                                                      float* __restrict__ fstage, uint64_t* bar, int lane) {
    uint32_t id[BATCH / 32];
#pragma unroll
    for (int k = 0; k < BATCH / 32; ++k) {
        const int r = k * 32 + lane;
        id[k] = (r < cnt) ? source_id(src, p0 + r) : 0u;
    }
#pragma unroll
    for (int k = 0; k < BATCH / 32; ++k) {
        const int r = k * 32 + lane;
        if (r < cnt) {
            const float* g = src.base + (size_t)id[k] * REC;
            const uint32_t d = smem_u32(stage + r * REC);
            cp_async16(d, g);
            cp_async16(d + 16u, g + 4);
            cp_async16(d + 32u, g + 8);
            cp_async16(smem_u32(fstage + r * FCH), fsrc + (size_t)id[k] * stride);
        }
    }
    cp_async_mbar_arrive_noinc(bar);
}

struct FeatState {
    F2 nA;              // -alpha_accum (a pixel outside the image starts saturated and never contributes)
    F2 f[FCH];          // sum of w * F[., c]
    uint32_t badbits;   // sticky: the exact-division range was left
    bool bad;           // sticky: some blend weight needs the double-precision expression
};

// fwd_walk (gsr_render.cu) without marks, depth or statistics, blending the FCH staged features instead of the colour
template <bool CHECK>
__device__ __forceinline__ void feat_walk(const float4* __restrict__ rec4, const float4* __restrict__ feat4,
                                          uint32_t list_addr, uint32_t dummy_addr, int my_cnt, int iters, F2 fpx,
                                          float fpy, FeatState& st) {
    const float neg_sat = -GSR_SAT_THRESH;
    for (int t = 0; t < iters; ++t) {
        const bool act = t < my_cnt;
        const int j = (int)lds_u8(act ? list_addr + t : dummy_addr);
        const float4 q0 = rec4[j * 3 + 0];
        const float4 q1 = rec4[j * 3 + 1];
        const float4 q2 = rec4[j * 3 + 2];
        const F2 du = add2(fpx, bc(-q0.x));
        const float dv = __fsub_rn(fpy, q0.y);
        const F2 t1 = mul2(du, bc(q1.y));
        const F2 t2 = mul2(du, bc(q1.z));
        const F2 t3n = mul2(t1, bc(-dv));
        const F2 t4 = fma2(du, t2, t3n);
        const float t5 = __fmul_rn(dv, q1.x);
        const F2 num = fma2(bc(dv), bc(t5), t4);
        st.badbits |= (__float_as_uint(lo(num)) - 0x1e000000u) | (__float_as_uint(hi(num)) - 0x1e000000u);
        const F2 q = mul2(num, bc(q2.x));
        const F2 r = fma2(bc(-q1.w), q, num);
        const F2 mh = fma2(bc(q2.x), r, q);
        const F2 xe = mul2(mul2(mh, bc(-0.5f)), bc(LOG2E_F));
        const F2 al = mul2(pk(ex2_ftz(lo(xe)), ex2_ftz(hi(xe))), bc(q0.w));
        const bool c0 = act & (lo(st.nA) >= neg_sat) & (lo(mh) > 0.0f) & (lo(al) > GSR_ALPHA_SKIP_MAX);
        const bool c1 = act & (hi(st.nA) >= neg_sat) & (hi(mh) > 0.0f) & (hi(al) > GSR_ALPHA_SKIP_MAX);
        const F2 alm = pk(c0 ? lo(al) : 0.0f, c1 ? hi(al) : 0.0f);
        const F2 w = fma2(st.nA, alm, alm);
        if (CHECK) {
            const F2 d = rsub2(w, alm);
            const F2 e = fma2(st.nA, alm, d);
            st.bad |= blend_hazard(lo(e), lo(w)) | blend_hazard(hi(e), hi(w));
        }
        st.nA = rsub2(w, st.nA);
        const float4 f = feat4[j];
        st.f[0] = fma2(w, bc(f.x), st.f[0]);
        st.f[1] = fma2(w, bc(f.y), st.f[1]);
        st.f[2] = fma2(w, bc(f.z), st.f[2]);
        st.f[3] = fma2(w, bc(f.w), st.f[3]);
    }
}

// exact_pixel (gsr_render.cu) for the features: one flagged pixel, start to end, with the reference's arithmetic
// (IEEE division, double-precision blend weight), by the whole warp; every lane returns the pixel's FCH sums
__device__ __noinline__ float4 feature_pixel_exact_warp(const RecSource src, const float* __restrict__ fsrc, int stride,
                                                        int start, int total, float fpx, float fpy, int lane) {
    float A = 0.0f, s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
    bool stop = false;
    for (int base = 0; base < total && !stop; base += 32) {
        const int i = base + lane;
        float alpha = 0.0f;
        float4 f = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (i < total) {
            const size_t row = (size_t)source_id(src, start + i);
            const float4* q = reinterpret_cast<const float4*>(src.base + row * REC);
            const float4 q0 = __ldg(q), q1 = __ldg(q + 1);
            const float du = __fsub_rn(fpx, q0.x), dv = __fsub_rn(fpy, q0.y);
            const float t1 = __fmul_rn(du, q1.y);
            const float t2 = __fmul_rn(du, q1.z);
            const float t4 = __fmaf_rn(du, t2, -__fmul_rn(dv, t1));
            const float num = __fmaf_rn(dv, __fmul_rn(dv, q1.x), t4);
            const float mh = __fdiv_rn(num, q1.w);
            if (mh > 0.0f) alpha = __fmul_rn(ex2_ftz(__fmul_rn(__fmul_rn(mh, -0.5f), LOG2E_F)), q0.w);
            if (alpha <= GSR_ALPHA_SKIP_MAX) alpha = 0.0f;
            f = __ldg(reinterpret_cast<const float4*>(fsrc + row * stride));
        }
        const int m = min(32, total - base);
        for (int k = 0; k < m; ++k) {
            if (A > GSR_SAT_THRESH) {
                stop = true;
                break;
            }
            const float ak = __shfl_sync(0xffffffffu, alpha, k);
            if (ak == 0.0f) continue;
            const float w = (float)((1.0 - (double)A) * (double)ak);
            A = __fadd_rn(A, w);
            s0 = __fmaf_rn(w, __shfl_sync(0xffffffffu, f.x, k), s0);
            s1 = __fmaf_rn(w, __shfl_sync(0xffffffffu, f.y, k), s1);
            s2 = __fmaf_rn(w, __shfl_sync(0xffffffffu, f.z, k), s2);
            s3 = __fmaf_rn(w, __shfl_sync(0xffffffffu, f.w, k), s3);
        }
    }
    return make_float4(s0, s1, s2, s3);
}

__global__ void __launch_bounds__(CTA_THREADS, GSR_FEAT_FWD_MINB)
    k_features_fwd(const RecSource rs, const int32_t* __restrict__ ranges, const float* __restrict__ features,
                   int stride, int D, int W, int H, float* __restrict__ feature_map) {
    __shared__ __align__(128) float s_rec[STAGES][BATCH * REC];
    __shared__ __align__(16) float s_feat[STAGES][BATCH * FCH];
    __shared__ __align__(8) uint64_t s_full[STAGES];
    __shared__ int s_cnt[STAGES];
    __shared__ __align__(16) uint8_t s_list[CTA_WARPS][LIST_BYTES];

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
    const int c0 = blockIdx.z * FCH;
    const float* fsrc = features + c0;
    const int start = ranges[tile];
    const int total = ranges[tile + 1] - start;
    const PixelMap pm = pixel_map(warp, lane);
    const int px = pm.px, py = pm.py;
    const bool valid0 = (px < W) && (py < H), valid1 = (px + 1 < W) && (py < H);
    const F2 fpx = pk((float)px, (float)(px + 1));
    const float fpy = (float)py;
    uint8_t* list = &s_list[warp][0];
    const uint32_t list_addr = smem_u32(list + (lane / GROUP_LANES) * BATCH);
    const uint32_t dummy_addr = smem_u32(list + LIST_DUMMY);
    if (lane == 0) list[LIST_DUMMY] = 0;

    const int nb = (total + BATCH - 1) / BATCH;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&s_full[s], 32);
            s_cnt[s] = 0;
        }
        fence_mbar_init();
    }
    __syncthreads();
    auto load_batch = [&](int b) {
        const int s = b % STAGES;
        gather_batch_features(rs, fsrc, stride, start + b * BATCH, min(BATCH, total - b * BATCH), &s_rec[s][0],
                              &s_feat[s][0], &s_full[s], lane);
    };
    if (warp == 0) {
        const int pre = nb < STAGES ? nb : STAGES;
        for (int b = 0; b < pre; ++b) load_batch(b);
    }

    FeatState st;
    st.nA = pk(valid0 ? -0.0f : -1.0f, valid1 ? -0.0f : -1.0f);
#pragma unroll
    for (int c = 0; c < FCH; ++c) st.f[c] = bc(0.0f);
    st.badbits = 0u;
    st.bad = false;
    const float neg_sat = -GSR_SAT_THRESH;

    for (int b = 0; b < nb; ++b) {
        const int s = b % STAGES;
        mbar_wait(&s_full[s], (uint32_t)((b / STAGES) & 1));
        const bool live0 = lo(st.nA) >= neg_sat, live1 = hi(st.nA) >= neg_sat;
        if (__any_sync(0xffffffffu, live0 || live1)) {
            const int cnt = min(BATCH, total - b * BATCH);
            const float4* rec4 = reinterpret_cast<const float4*>(&s_rec[s][0]);
            const float4* feat4 = reinterpret_cast<const float4*>(&s_feat[s][0]);
            int cnts[GROUPS];
            st.bad |= build_lists<true>(rec4, cnt, lane, pm.bx0, pm.by0, list, cnts);
            const int my_cnt = group_select(cnts, lane / GROUP_LANES);
            const int iters = group_max(cnts);
            const bool small = (live0 && lo(st.nA) > -0.015625f) || (live1 && hi(st.nA) > -0.015625f);
            if (__any_sync(0xffffffffu, small))
                feat_walk<true>(rec4, feat4, list_addr, dummy_addr, my_cnt, iters, fpx, fpy, st);
            else
                feat_walk<false>(rec4, feat4, list_addr, dummy_addr, my_cnt, iters, fpx, fpy, st);
        }
        if (stage_checkout(&s_cnt[s], lane) && b + STAGES < nb) load_batch(b + STAGES);
    }

    float v0[FCH], v1[FCH];
#pragma unroll
    for (int c = 0; c < FCH; ++c) {
        v0[c] = lo(st.f[c]);
        v1[c] = hi(st.f[c]);
    }
    const bool bad = st.bad || (st.badbits & 0xc0000000u) != 0u;
    uint32_t todo = __ballot_sync(0xffffffffu, bad && valid0);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int sx = __shfl_sync(0xffffffffu, px, src), sy = __shfl_sync(0xffffffffu, py, src);
        const bool two = __shfl_sync(0xffffffffu, valid1 ? 1 : 0, src) != 0;
        const float4 e0 = feature_pixel_exact_warp(rs, fsrc, stride, start, total, (float)sx, (float)sy, lane);
        if (lane == src) { v0[0] = e0.x; v0[1] = e0.y; v0[2] = e0.z; v0[3] = e0.w; }
        if (two) {
            const float4 e1 = feature_pixel_exact_warp(rs, fsrc, stride, start, total, (float)(sx + 1), (float)sy, lane);
            if (lane == src) { v1[0] = e1.x; v1[1] = e1.y; v1[2] = e1.z; v1[3] = e1.w; }
        }
    }
    const int nc = min(FCH, D - c0);
    if (valid0) {
        float* o = feature_map + ((size_t)py * W + px) * D + c0;
#pragma unroll
        for (int c = 0; c < FCH; ++c)
            if (c < nc) o[c] = v0[c];
    }
    if (valid1) {
        float* o = feature_map + ((size_t)py * W + px + 1) * D + c0;
#pragma unroll
        for (int c = 0; c < FCH; ++c)
            if (c < nc) o[c] = v1[c];
    }
}

// MASKS: the per-group lists come from the colour forward's contribution masks, else from the footprint test (then a
// step nobody in the warp contributes to is skipped, as in k_render_bwd)
template <bool MASKS>
__global__ void __launch_bounds__(CTA_THREADS, GSR_FEAT_BWD_MINB)
    k_features_bwd(const RecSource rs, const int32_t* __restrict__ ranges, int W, int H,
                   const int32_t* __restrict__ n_in, const float* __restrict__ w_in,
                   const float* __restrict__ features, int stride, int D, const float* __restrict__ grad_map,
                   float* __restrict__ grad_features, float* __restrict__ grad_rows,
                   const uint32_t* __restrict__ masks) {
    __shared__ __align__(128) float s_rec[BSTAGES][(BATCH + 1) * REC];  // + an all-zero record (alpha 0) per stage
    __shared__ __align__(16) float s_feat[BSTAGES][(BATCH + 1) * FCH];
    __shared__ __align__(8) uint64_t s_full[BSTAGES];
    __shared__ int s_cnt[BSTAGES];
    __shared__ float s_acc[BSTAGES][BATCH * NGF];
    __shared__ __align__(16) uint8_t s_list[CTA_WARPS][LIST_BYTES];
    __shared__ int s_maxn;

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
    const int c0 = blockIdx.z * FCH;
    const float* fsrc = features + c0;
    const int start = ranges[tile];
    const PixelMap pm = pixel_map(warp, lane);
    const int px = pm.px, py = pm.py;
    const bool valid0 = (px < W) && (py < H), valid1 = (px + 1 < W) && (py < H);
    const F2 fpx = pk((float)px, (float)(px + 1));
    const float fpy = (float)py;
    uint8_t* list = &s_list[warp][0];
    const uint32_t list_addr = smem_u32(list + (lane / GROUP_LANES) * BATCH);
    const uint32_t dummy_addr = smem_u32(list + LIST_DUMMY);
    if (lane == 0) list[LIST_DUMMY] = (uint8_t)BATCH;  // -> the all-zero record
    const uint32_t* gm = MASKS ? masks + ((size_t)(start / BATCH + tile) * MASK_WORDS_PER_SLOT + warp * GROUPS * MASK_WORDS)
                               : nullptr;

    const int nc = min(FCH, D - c0);
    int n0 = 0, n1 = 0;
    float wt0 = 0.0f, wt1 = 0.0f, ga[FCH], gb[FCH];
#pragma unroll
    for (int c = 0; c < FCH; ++c) ga[c] = gb[c] = 0.0f;
    if (valid0) {
        const size_t pix = (size_t)py * W + px;
        n0 = n_in[pix];
        wt0 = w_in[pix];
#pragma unroll
        for (int c = 0; c < FCH; ++c)
            if (c < nc) ga[c] = grad_map[pix * D + c0 + c];
    }
    if (valid1) {
        const size_t pix = (size_t)py * W + px + 1;
        n1 = n_in[pix];
        wt1 = w_in[pix];
#pragma unroll
        for (int c = 0; c < FCH; ++c)
            if (c < nc) gb[c] = grad_map[pix * D + c0 + c];
    }
    F2 weight = pk(wt0, wt1);
    F2 G[FCH];
#pragma unroll
    for (int c = 0; c < FCH; ++c) G[c] = pk(ga[c], gb[c]);
    if (tid == 0) {
        s_maxn = 0;
#pragma unroll
        for (int s = 0; s < BSTAGES; ++s) {
            mbar_init(&s_full[s], 32);
            s_cnt[s] = 0;
        }
        fence_mbar_init();
    }
    __syncthreads();
    {
        int m = max(n0, n1);
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 16));
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 8));
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 4));
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 2));
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 1));
        if (lane == 0) atomicMax(&s_maxn, m);
    }
    for (int k = tid; k < BSTAGES * BATCH * NGF; k += CTA_THREADS) (&s_acc[0][0])[k] = 0.0f;
    if (tid < BSTAGES * REC) s_rec[tid / REC][BATCH * REC + tid % REC] = 0.0f;
    if (tid < BSTAGES * FCH) s_feat[tid / FCH][BATCH * FCH + tid % FCH] = 0.0f;
    __syncthreads();
    const int total = s_maxn;  // deepest splat any pixel of this tile consumed
    const int nb = (total + BATCH - 1) / BATCH;
    if (nb == 0) return;

    auto load_slot = [&](int k) {
        const int b = nb - 1 - k, s = k % BSTAGES;
        gather_batch_features(rs, fsrc, stride, start + b * BATCH, min(BATCH, total - b * BATCH), &s_rec[s][0],
                              &s_feat[s][0], &s_full[s], lane);
    };
    if (warp == 0) {
        const int pre = nb < BSTAGES ? nb : BSTAGES;
        for (int k = 0; k < pre; ++k) load_slot(k);
    }

    F2 na[FCH];  // -feature_accum
#pragma unroll
    for (int c = 0; c < FCH; ++c) na[c] = bc(-0.0f);
    const int gl = lane % GROUP_LANES;
    const uint32_t group_mask = 0xffu << (lane & ~(GROUP_LANES - 1));

    for (int k = 0; k < nb; ++k) {
        const int b = nb - 1 - k;
        const int s = k % BSTAGES;
        const int cnt = min(BATCH, total - b * BATCH);
        mbar_wait(&s_full[s], (uint32_t)((k / BSTAGES) & 1));
        const float4* rec4 = reinterpret_cast<const float4*>(&s_rec[s][0]);
        const float4* feat4 = reinterpret_cast<const float4*>(&s_feat[s][0]);
        float* acc = &s_acc[s][0];
        uint32_t acc_cell = smem_u32(acc) + gl * 4;  // this lane's moment cell of record 0
        asm volatile("" : "+r"(acc_cell));
        int cnts[GROUPS];
        if (MASKS)
            mask_lists(gm + (size_t)b * MASK_WORDS_PER_SLOT, cnt, lane, list, cnts);
        else
            build_lists(rec4, cnt, lane, pm.bx0, pm.by0, list, cnts);
        const int my_cnt = group_select(cnts, lane / GROUP_LANES);
        const int iters = group_max(cnts);
        const int chunk_base1 = (b * BATCH) % CHUNK_REF + 1;
        int base_idx = b * BATCH;
        asm volatile("" : "+r"(base_idx));

        for (int step = 0; step < iters; ++step) {
            const int tt = my_cnt - 1 - step;
            const bool act = tt >= 0;
            const int j = (int)lds_u8(act ? list_addr + tt : dummy_addr);
            const int idx = base_idx + j;
            // the colour backward's per-(pixel, splat) arithmetic up to d_alpha (render_bwd in gsr_render.cu)
            const float4 q0 = rec4[j * 3 + 0];
            const float4 q1 = rec4[j * 3 + 1];
            const float4 q2 = rec4[j * 3 + 2];
            const float rdet = q2.x, opa = q0.w;
            const F2 du = add2(fpx, bc(-q0.x));
            const float dv = __fsub_rn(fpy, q0.y);
            const F2 s1 = mul2(du, mul2(du, bc(q1.z)));
            const float s3 = __fmul_rn(dv, __fmul_rn(dv, q1.x));
            const F2 s12 = fma2(bc(-dv), mul2(du, bc(q1.y)), s1);
            const F2 mh = mul2(add2(s12, bc(s3)), bc(rdet));
            const F2 xe = mul2(mul2(mh, bc(-0.5f)), bc(LOG2E_F));
            const float g0 = lo(mh) > 0.0f ? ex2_ftz(lo(xe)) : 0.0f;
            const float g1 = hi(mh) > 0.0f ? ex2_ftz(hi(xe)) : 0.0f;
            const F2 og = mul2(pk(g0, g1), bc(opa));
            const float al0 = fminf(GSR_ALPHA_CLAMP, lo(og));
            const float al1 = fminf(GSR_ALPHA_CLAMP, hi(og));
            const bool c0p = (idx < n0) & (al0 > GSR_ALPHA_SKIP_MAX);
            const bool c1p = (idx < n1) & (al1 > GSR_ALPHA_SKIP_MAX);
            const uint32_t bal = MASKS ? 0xffffffffu : __ballot_sync(0xffffffffu, c0p | c1p);
            if (!MASKS && bal == 0u) continue;
            const F2 alpha = pk(c0p ? al0 : 0.0f, c1p ? al1 : 0.0f);
            const F2 gmv = pk(c0p ? g0 : 0.0f, c1p ? g1 : 0.0f);
            const F2 r = recip_one_minus2(alpha);
            int local1 = chunk_base1 + j;
            if (local1 > CHUNK_REF) local1 -= CHUNK_REF;
            const F2 wr = mul2(weight, r);
            weight = pk((c0p & (local1 < n0)) ? lo(wr) : lo(weight), (c1p & (local1 < n1)) ? hi(wr) : hi(weight));
            // t_c = weight*f_c - r*acc_c ; d_alpha = sum_c G_c * t_c ; acc_c += weight * (alpha * f_c)
            const float4 f = feat4[j];
            const float fv[FCH] = {f.x, f.y, f.z, f.w};
            F2 galpha = bc(0.0f);
#pragma unroll
            for (int c = 0; c < FCH; ++c) {
                const F2 tc = fma2(weight, bc(fv[c]), mul2(r, na[c]));
                galpha = fma2(G[c], tc, galpha);
                na[c] = fma2(weight, mul2(alpha, bc(-fv[c])), na[c]);
            }
            const F2 aw = mul2(alpha, weight);
            const F2 gmh = mul2(mul2(gmv, bc(-0.5f)), mul2(bc(opa), galpha));
            const F2 hu = mul2(gmh, du), hv = mul2(gmh, bc(dv));
            float g8[8];
#pragma unroll
            for (int c = 0; c < FCH; ++c) {
                const F2 mf = mul2(G[c], aw);
                g8[c] = lo(mf) + hi(mf);
            }
            const F2 m3 = mul2(galpha, gmv), m6 = mul2(hu, du), m7 = mul2(hu, bc(dv)), m8 = mul2(hv, bc(dv));
            g8[4] = lo(m3) + hi(m3);
            g8[5] = lo(hu) + hi(hu);
            g8[6] = lo(hv) + hi(hv);
            g8[7] = lo(m6) + hi(m6);
            float t4[4] = {lo(m7) + hi(m7), lo(m8) + hi(m8), 0.0f, 0.0f};
            // lane gl of the group ends with moment gl (0..7), lanes 0 and 1 also with moments 8 and 9
            butterfly8_quarter(g8, lane);
            butterfly4_quarter_low(t4, lane);
            const bool group_any = MASKS ? act : ((bal & group_mask) != 0u);
            if (group_any) {
                float* cell = reinterpret_cast<float*>(__cvta_shared_to_generic(acc_cell + j * (NGF * 4)));
                atomicAdd(cell, g8[0]);
                if (gl < 2) atomicAdd(cell + 8, t4[0]);
            }
        }
        // the last warp to leave the batch flushes its records' moments (one v4 reduction of feature gradients, the
        // geometry finished as in k_render_bwd and added into the rows' slots 3..8), clears them and recycles the stage
        if (stage_checkout(&s_cnt[s], lane)) {
            int gids[BATCH / 32];
#pragma unroll
            for (int i = 0; i < BATCH / 32; ++i) {
                const int r = lane + 32 * i;
                gids[i] = (r >= cnt) ? 0 : (int)source_id(rs, start + b * BATCH + r);
            }
#pragma unroll
            for (int i = 0; i < BATCH / 32; ++i) {
                const int r = lane + 32 * i;
                if (r >= cnt) break;
                float S[NGF];
                bool any = false;
#pragma unroll
                for (int q = 0; q < NGF; ++q) {
                    S[q] = acc[r * NGF + q];
                    any |= (S[q] != 0.0f);
                }
                if (any) {
#pragma unroll
                    for (int q = 0; q < NGF; ++q) acc[r * NGF + q] = 0.0f;
                    const float4 q1 = rec4[r * 3 + 1];
                    const float a = q1.x, bh = 0.5f * q1.y, c = q1.z, rdet = rec4[r * 3 + 2].x;
                    const size_t gid = (size_t)gids[i];
                    red_add_v4(grad_features + gid * stride + c0, S[0], S[1], S[2], S[3]);
                    const float gu = -rdet * (2.0f * c * S[5] - 2.0f * bh * S[6]);
                    const float gv = -rdet * (2.0f * a * S[6] - 2.0f * bh * S[5]);
                    const float cf = (a * S[9] - 2.0f * bh * S[8] + c * S[7]) * rdet * rdet;
                    const float gc0 = -c * cf + S[9] * rdet, gc1 = bh * cf - S[8] * rdet, gc2 = -a * cf + S[7] * rdet;
                    float* row = grad_rows + gid * GRAD_ROW;
                    atomicAdd(row + 3, S[4]);
                    red_add_v4(row + 4, gu, gv, gc0, gc1);
                    atomicAdd(row + 8, gc2);
                }
            }
            __syncwarp();
            if (k + BSTAGES < nb) {
                __threadfence_block();  // every lane: its share of the cleared accumulator before its arrival
                load_slot(k + BSTAGES);
            }
        }
    }
}

}  // namespace gsr

using namespace gsr;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// the arguments both entry points share
static bool features_args_ok(const float* records, const uint64_t* keys_sorted, const int32_t* ids_sorted,
                             const int32_t* ranges, int H, int W, const float* features, int stride, int D) {
    if ((keys_sorted == nullptr) == (ids_sorted == nullptr)) return false;  // exactly one id source
    if (records == nullptr || ranges == nullptr || features == nullptr || !aligned16(features)) return false;
    if (H <= 0 || W <= 0 || D <= 0) return false;
    if (stride % FCH != 0 || stride < D || stride >= D + FCH || stride / FCH > 65535) return false;
    return true;
}

extern "C" {

int gsr_render_features_forward(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                                const int32_t* ids_sorted, const int32_t* ranges, int H, int W, const float* features,
                                int feature_stride, int D, float* feature_map, void* stream) {
    if (!features_args_ok(gaussian_records, keys_sorted, ids_sorted, ranges, H, W, features, feature_stride, D) ||
        feature_map == nullptr)
        return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE, feature_stride / FCH), block(CTA_THREADS);
    k_features_fwd<<<grid, block, 0, (cudaStream_t)stream>>>(
        make_source(gaussian_records, keys_sorted, ids_sorted, id_bits), ranges, features, feature_stride, D, W, H,
        feature_map);
    return (int)cudaGetLastError();
}

int gsr_render_features_backward(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                                 const int32_t* ids_sorted, const int32_t* ranges, int H, int W, const int32_t* n_in,
                                 const float* w_in, const float* features, int feature_stride, int D,
                                 const float* grad_feature_map, float* grad_features, float* grad_rows,
                                 const uint32_t* contribution_masks, void* stream) {
    if (!features_args_ok(gaussian_records, keys_sorted, ids_sorted, ranges, H, W, features, feature_stride, D))
        return GSR_ERR_BAD_ARG;
    if (n_in == nullptr || w_in == nullptr || grad_feature_map == nullptr || grad_features == nullptr ||
        grad_rows == nullptr || !aligned16(grad_features) || !aligned16(grad_rows))
        return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE, feature_stride / FCH), block(CTA_THREADS);
    const RecSource src = make_source(gaussian_records, keys_sorted, ids_sorted, id_bits);
    cudaStream_t st = (cudaStream_t)stream;
    if (contribution_masks != nullptr)
        k_features_bwd<true><<<grid, block, 0, st>>>(src, ranges, W, H, n_in, w_in, features, feature_stride, D,
                                                     grad_feature_map, grad_features, grad_rows, contribution_masks);
    else
        k_features_bwd<false><<<grid, block, 0, st>>>(src, ranges, W, H, n_in, w_in, features, feature_stride, D,
                                                      grad_feature_map, grad_features, grad_rows, nullptr);
    return (int)cudaGetLastError();
}

}  // extern "C"
