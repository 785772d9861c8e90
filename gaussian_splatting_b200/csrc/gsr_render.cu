// gsr_render.cu — fp32 tile renderers (forward + backward), one CTA per 16x16 tile.
//
// Contract (values): src/render.cu:101-188 and src/render_backward.cu:120-284 of the
// reference, fp32 branch (use_fast_exp): +0.25 dilation, __expf, alpha < 1/255 skip,
// saturation early-out at 0.9999, background blend below 0.999, and the backward's
// chunk-local weight recurrence (SURVEY.md Q2-Q10).  The forward is BIT-EXACT with
// the reference build: the inner loop issues the same rounded operations in the same
// order (read off the reference's SASS, DESIGN.md "Rounding contract").
//
// Structure (what is different from the reference):
//   * input is the per-gaussian array of 48-byte records, read in depth order through the sorted pair list;
//     batches of BATCH records are staged into a shared-memory ring by 16-byte cp.async copies completing on
//     an mbarrier, instead of 256 threads gathering 4-byte fields through an index array.  Stages are recycled
//     at WARP granularity (stage_checkout): the last warp to leave a stage re-arms it and fetches the next
//     batch, there is no CTA-wide barrier in either batch loop;
//   * a CTA is 128 threads; a lane carries TWO horizontally adjacent pixels and evaluates them as pairs of
//     scalar IEEE operations (gsr_f32x2.cuh; du is a pixel pair, dv and all per-splat constants are shared by
//     both halves), so the per-splat work of a lane is paid once for two pixels;
//   * a warp owns a 16x4 pixel band, each HALF-warp an 8x4 block.  For every batch the warp tests each
//     record's "cannot contribute" bound (gsr_record.cuh) against both blocks, 4 records per lane, and
//     compacts the survivors into one index list per half-warp in shared memory; the two halves then walk
//     their own lists side by side, so one instruction stream evaluates two different splats.  A culled
//     splat would have been skipped by the reference's alpha < 1/255 test for all 32 pixels, so results do
//     not change — per-pixel evaluations drop to ~34% of (pixels x splats of the tile);
//   * the division num/det uses the record's correctly rounded reciprocal (3 packed FMAs, still the
//     correctly rounded IEEE quotient) instead of MUFU.RCP + 5 FMAs + FCHK per pixel;
//   * the forward walk is one branch-free basic block; the two rare events that need slow exact
//     arithmetic only raise sticky flags and the flagged pixels are recomputed afterwards by the whole warp;
//   * per-pixel colour lives in registers (reference: shared-memory image tile);
//   * a warp whose 64 pixels are saturated passes the remaining batches on without touching them
//     (reference walks every chunk of the tile);
//   * backward: starts at the deepest splat any pixel of the tile actually used; the 9 partial
//     derivatives of a (half-warp, splat) are reduced with a value-splitting butterfly (12 shuffles
//     instead of 45), combined across the warps in a per-stage shared-memory accumulator, and ONE set of 9
//     atomics per (gaussian, tile) pair goes to HBM (reference: 72 unconditional atomics), issued by the
//     warp that recycles the stage.
#include "gsr_tile_walk.cuh"

namespace gsr {

#ifdef GSR_STATS
__device__ unsigned long long g_stats[16];  // 0..7 forward, 8..15 backward
#define STAT(i, v) atomicAdd(&g_stats[i], (unsigned long long)(v))
#else
#define STAT(i, v)
#endif
// ---------------------------------------------------------------------------------------------------
// Forward.  The inner loop is ONE basic block (no branches): rare events that need the slow exact
// arithmetic only raise a sticky per-pixel flag, and a flagged pixel is recomputed from scratch by
// render_pixel_exact_warp() after the walk.  Two such events exist:
//   (1) division: q = num*rcp; q += rcp*fma(-det,q,num) is the correctly rounded num/det only for
//       |num| in [2^-67, 2^61) and records whose 1/det could be refined (rcp != 0);
//   (2) blend weight: the reference evaluates w = (float)((1.0 - (double)A) * (double)alpha)
//       (src/render.cu:147-148).  (1 - A)*alpha = alpha - A*alpha is exact in double whenever A == 0 or
//       A >= 2^-6 (1 - A then has at most 29 significant bits), so ONE fp32 FMA returns the same float.  For
//       0 < A < 2^-6 the double product itself rounds at 53 bits, and the two roundings differ from the FMA's
//       one only if the exact value lies within 2^-53 (relative) of a rounding midpoint; then the FMA's
//       residual e = RN(alpha - A*alpha - w) is exactly +-half an ulp of w, i.e. a power of two.  The walk
//       is compiled twice: while some live pixel of the warp still has A < 2^-6 the CHECK version computes
//       e (two more packed operations) and flags the pixel when |e| is half (or a quarter of) an ulp of w
//       (about one blend in 2^23); afterwards the plain version runs.
struct FwdState {
    F2 nA;        // -alpha_accum (a pixel outside the image starts saturated and never contributes)
    F2 wl;        // alpha_weight of the last contributing splat
    F2 C0, C1, C2;
    F2 D;               // depth/alpha mode: sum of w * z (unused otherwise)
    int last0, last1;   // tile index + 1 of the last contributing splat (0: none)
    uint32_t badbits;   // sticky: top two bits set <=> some numerator left the exact-division range
    bool bad;           // sticky: some blend weight needs the double-precision expression
};

__device__ __forceinline__ void sts_u8(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// Blend-weight statistics (GSR weight_stats, DESIGN.md 3.14): per gaussian, over the pixels it contributes to,
// sum w, max w and the number of such pixels, w the weight of the colour blend.  Destinations are per-gaussian rows
// accumulated into; pair_total / capacity guard the speculatively sized pair buffers: when the scan's pair count
// (low 32 bits of *pair_total) exceeds the capacity the kernel ran with, its output is discarded by the host and
// nothing is added.
struct WeightSink {
    float* sum;
    uint32_t* max;              // float bits; w >= +0 so the unsigned order is the float order
    uint32_t* count;
    const uint64_t* pair_total; // NULL: no guard
    uint32_t capacity;
};
// Per-stage shared accumulator WeightAcc: [sum (f32 bits) | max | count] x BATCH words, indexed by staged record.
constexpr int WACC_WORDS = 3 * BATCH;

// One walk step: the lane group's 16 pixels reduced (xor shuffles within the group, ballots for the count), one
// lane per group adds into the record's accumulator.  The sum goes through a shared fp32 atomicAdd (a CAS loop on
// sm_90); it is issued only by groups where record j contributed.
__device__ __forceinline__ void weight_stats_step(uint32_t* __restrict__ wacc, int j, F2 w, bool c0, bool c1,
                                                  int lane) {
    float s = lo(w) + hi(w);
    uint32_t m = max(__float_as_uint(lo(w)), __float_as_uint(hi(w)));
#pragma unroll
    for (int o = GROUP_LANES / 2; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    const uint32_t gmask = ((1u << GROUP_LANES) - 1u) << (lane & ~(GROUP_LANES - 1));
    const uint32_t n = __popc(__ballot_sync(0xffffffffu, c0) & gmask) + __popc(__ballot_sync(0xffffffffu, c1) & gmask);
    if ((lane % GROUP_LANES) == 0 && n != 0u) {
        atomicAdd(reinterpret_cast<float*>(wacc + j), s);
        atomicMax(wacc + BATCH + j, m);
        atomicAdd(wacc + 2 * BATCH + j, n);
    }
}

// By the warp that checked the stage out last: every staged record with a non-zero count goes to HBM (three
// reductions), and its accumulator is cleared for the stage's next batch.  The caller orders the clearing stores
// before the stage is re-armed (__threadfence_block ahead of the refill's arrivals), as the backward does.
__device__ __forceinline__ void weight_stats_flush(uint32_t* __restrict__ wacc, const RecSource& src, int p0, int cnt,
                                                   const WeightSink& ws, int lane) {
    const bool keep = ws.pair_total == nullptr || (uint32_t)__ldg(ws.pair_total) <= ws.capacity;
#pragma unroll
    for (int k = 0; k < BATCH / 32; ++k) {
        const int r = k * 32 + lane;
        if (r >= cnt) break;
        const uint32_t n = wacc[2 * BATCH + r];
        if (n == 0u) continue;
        const float s = __uint_as_float(wacc[r]);
        const uint32_t m = wacc[BATCH + r];
        wacc[r] = wacc[BATCH + r] = wacc[2 * BATCH + r] = 0u;
        if (keep) {
            const uint32_t id = source_id(src, p0 + r);
            atomicAdd(ws.sum + id, s);
            atomicMax(ws.max + id, m);
            atomicAdd(ws.count + id, n);
        }
    }
}

// MARK: the walk also records, per lane group, WHICH staged records contributed to at least one pixel of the group.
// Inside the loop the marks are list positions in a register — a store inside the loop costs ptxas's register-pair
// coalescing (+11 instructions per iteration, measured) — so the walk is split into runs of 32 positions and the
// inner loop stays one basic block.  After each run the positions are OR-reduced over each group and lane l turns
// position t0 + l of every group into a byte flag per record (flag_addr: this warp's [GROUPS][BATCH] bytes, zero on
// entry); after the walk one ballot per 32 records turns the flags into the group's 128-bit record mask, stored to
// gm_warp[group][word], and the flags are cleared again.
// DEPTH: also D += w * z, z from the stage's z array zs (same weight w as the colour blend).
// STATS: also the blend-weight statistics of every walked record (WeightAcc: the stage's accumulator wacc).
template <bool CHECK, bool MARK, bool DEPTH = false, bool STATS = false>
__device__ __forceinline__ void fwd_walk(const float4* __restrict__ rec4, uint32_t list_addr, uint32_t dummy_addr,
                                         int my_cnt, int iters, int next_base, F2 fpx, float fpy, FwdState& st,
                                         uint32_t* __restrict__ gm_warp, uint32_t flag_addr, int lane,
                                         const float* __restrict__ zs = nullptr, uint32_t* __restrict__ wacc = nullptr) {
    const float neg_sat = -GSR_SAT_THRESH;
    int lj0 = -1, lj1 = -1;  // record (within this batch) of the last contribution
    for (int t0 = 0; t0 < iters; t0 += (MARK ? 32 : BATCH)) {
    const int t_end = MARK ? min(iters, t0 + 32) : iters;
    uint32_t pmask = 0u, pbit = 1u;
#pragma unroll FWD_UNROLL
    for (int t = t0; t < t_end; ++t) {
        const bool act = t < my_cnt;
        const int j = (int)lds_u8(act ? list_addr + t : dummy_addr);
        const float4 q0 = rec4[j * 3 + 0];  // u v tau opacity
        const float4 q1 = rec4[j * 3 + 1];  // a 2b c det
        const float4 q2 = rec4[j * 3 + 2];  // rcp colour
        // Mahalanobis numerator c*du*du - (b+b)*du*dv + a*dv*dv, reference rounding order
        // (src/render.cu:130-131); dv is shared by the pair
        const F2 du = add2(fpx, bc(-q0.x));
        const float dv = __fsub_rn(fpy, q0.y);
        const F2 t1 = mul2(du, bc(q1.y));
        const F2 t2 = mul2(du, bc(q1.z));
        const F2 t3n = mul2(t1, bc(-dv));
        const F2 t4 = fma2(du, t2, t3n);
        const float t5 = __fmul_rn(dv, q1.x);
        const F2 num = fma2(bc(dv), bc(t5), t4);
        // exact-division range check, sticky: x - 2^-67 (as bits) must stay below 2^30 * 2^23
        st.badbits |= (__float_as_uint(lo(num)) - 0x1e000000u) | (__float_as_uint(hi(num)) - 0x1e000000u);
        const F2 q = mul2(num, bc(q2.x));
        const F2 r = fma2(bc(-q1.w), q, num);
        const F2 mh = fma2(bc(q2.x), r, q);
        const F2 xe = mul2(mul2(mh, bc(-0.5f)), bc(LOG2E_F));
        const F2 al = mul2(pk(ex2_ftz(lo(xe)), ex2_ftz(hi(xe))), bc(q0.w));
        // contributes: pixel not saturated yet, mh > 0, alpha above the 1/255 skip
        // ((double)alpha < 0.00392156862 skips).  Bitwise & on purpose: no short-circuit branches here.
        const bool c0 = act & (lo(st.nA) >= neg_sat) & (lo(mh) > 0.0f) & (lo(al) > GSR_ALPHA_SKIP_MAX);
        const bool c1 = act & (hi(st.nA) >= neg_sat) & (hi(mh) > 0.0f) & (hi(al) > GSR_ALPHA_SKIP_MAX);
        const F2 alm = pk(c0 ? lo(al) : 0.0f, c1 ? hi(al) : 0.0f);
        const F2 w = fma2(st.nA, alm, alm);
        if (CHECK) {
            const F2 d = rsub2(w, alm);          // alpha - w, exact (Sterbenz) while A < 1/2
            const F2 e = fma2(st.nA, alm, d);
            st.bad |= blend_hazard(lo(e), lo(w)) | blend_hazard(hi(e), hi(w));
        }
        const F2 wnew = add2(bc(1.0f), st.nA);  // 1 - alpha_accum before this splat
        st.wl = pk(c0 ? lo(wnew) : lo(st.wl), c1 ? hi(wnew) : hi(st.wl));
        st.nA = rsub2(w, st.nA);
        st.C0 = fma2(w, bc(q2.y), st.C0);
        st.C1 = fma2(w, bc(q2.z), st.C1);
        st.C2 = fma2(w, bc(q2.w), st.C2);
        if (DEPTH) st.D = fma2(w, bc(zs[j]), st.D);
        if (STATS) weight_stats_step(wacc, j, w, c0, c1, lane);
        lj0 = c0 ? j : lj0;
        lj1 = c1 ? j : lj1;
        if (MARK) {
            pmask |= (c0 | c1) ? pbit : 0u;
            pbit <<= 1;
        }
    }
    if (MARK) {  // OR over each lane group (full-warp reductions: all groups execute the same instructions)
#pragma unroll
        for (int g = 0; g < GROUPS; ++g) {
            const uint32_t gsum = __reduce_or_sync(0xffffffffu, (lane / GROUP_LANES == g) ? pmask : 0u);
            if ((gsum >> lane) & 1u) {  // list position t0 + lane of group g contributed: flag its record
                const uint32_t j = lds_u8(list_addr + (g - lane / GROUP_LANES) * BATCH + t0 + lane);
                sts_u8(flag_addr + g * BATCH + j, 1u);
            }
        }
    }
    }
    if (MARK) {
        __syncwarp();
        uint32_t mine = 0u;
#pragma unroll
        for (int g = 0; g < GROUPS; ++g) {
#pragma unroll
            for (int w = 0; w < MASK_WORDS; ++w) {
                const uint32_t m = __ballot_sync(0xffffffffu, lds_u8(flag_addr + g * BATCH + w * 32 + lane) != 0u);
                mine = (lane == g * MASK_WORDS + w) ? m : mine;
            }
        }
        if (lane < GROUPS * MASK_WORDS) gm_warp[lane] = mine;
        __syncwarp();
        asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(flag_addr + lane * 16), "r"(0u) : "memory");
    }
    if (lj0 >= 0) st.last0 = next_base + lj0;
    if (lj1 >= 0) st.last1 = next_base + lj1;
}

// One pixel, start to end, with the reference's arithmetic spelled out (IEEE division, double-precision
// blend weight), computed by the WHOLE warp: lanes evaluate alpha of 32 consecutive splats in parallel,
// then every lane replays the (sequential) blend of those 32 from shuffles, so all lanes hold the same
// result.  Only runs for pixels flagged by the walk above (a handful per frame).
struct ExactPixel {
    float A, wl, c0, c1, c2;
    int n;
};
struct ExactPixelDepth {
    ExactPixel p;
    float d;  // sum of w * z, in the same order
};
template <bool DEPTH>
__device__ __forceinline__ ExactPixel exact_pixel(const RecSource& src, const DepthSource& ds, int start, int total,
                                                  float fpx, float fpy, int lane, float& d) {
    ExactPixel o;
    o.A = o.wl = o.c0 = o.c1 = o.c2 = 0.0f;
    o.n = total;
    d = 0.0f;
    bool stop = false;
    for (int base = 0; base < total && !stop; base += 32) {
        const int i = base + lane;
        float alpha = 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f, zi = 0.0f;
        if (i < total) {
            const size_t row = DEPTH ? (size_t)source_id_z(src, ds, start + i, zi) : (size_t)source_id(src, start + i);
            const float4* q = reinterpret_cast<const float4*>(src.base + row * REC);
            const float4 q0 = __ldg(q), q1 = __ldg(q + 1), q2 = __ldg(q + 2);
            const float du = __fsub_rn(fpx, q0.x), dv = __fsub_rn(fpy, q0.y);
            const float t1 = __fmul_rn(du, q1.y);
            const float t2 = __fmul_rn(du, q1.z);
            const float t4 = __fmaf_rn(du, t2, -__fmul_rn(dv, t1));
            const float num = __fmaf_rn(dv, __fmul_rn(dv, q1.x), t4);
            const float mh = __fdiv_rn(num, q1.w);
            if (mh > 0.0f) alpha = __fmul_rn(ex2_ftz(__fmul_rn(__fmul_rn(mh, -0.5f), LOG2E_F)), q0.w);
            if (alpha <= GSR_ALPHA_SKIP_MAX) alpha = 0.0f;
            cr = q2.y;
            cg = q2.z;
            cb = q2.w;
        }
        const int m = min(32, total - base);
        for (int k = 0; k < m; ++k) {
            if (o.A > GSR_SAT_THRESH) {  // tested before every splat of the tile list (src/render.cu:106)
                o.n = base + k;
                stop = true;
                break;
            }
            const float ak = __shfl_sync(0xffffffffu, alpha, k);
            if (ak == 0.0f) continue;
            const float w = (float)((1.0 - (double)o.A) * (double)ak);
            o.wl = __fsub_rn(1.0f, o.A);
            o.A = __fadd_rn(o.A, w);
            o.c0 = __fmaf_rn(w, __shfl_sync(0xffffffffu, cr, k), o.c0);
            o.c1 = __fmaf_rn(w, __shfl_sync(0xffffffffu, cg, k), o.c1);
            o.c2 = __fmaf_rn(w, __shfl_sync(0xffffffffu, cb, k), o.c2);
            if (DEPTH) d = __fmaf_rn(w, __shfl_sync(0xffffffffu, zi, k), d);
        }
    }
    return o;
}
__device__ __noinline__ ExactPixel render_pixel_exact_warp(const RecSource src, int start, int total, float fpx,
                                                           float fpy, int lane) {
    float d;
    return exact_pixel<false>(src, DepthSource{}, start, total, fpx, fpy, lane, d);
}
__device__ __noinline__ ExactPixelDepth render_pixel_exact_warp_depth(const RecSource src, const DepthSource ds,
                                                                      int start, int total, float fpx, float fpy,
                                                                      int lane) {
    ExactPixelDepth o;
    o.p = exact_pixel<true>(src, ds, start, total, fpx, fpy, lane, o.d);
    return o;
}

// MARK: also record, per (batch, warp, lane group), which staged records contributed (contribution masks for
// the backward; `masks` must be zero-filled by the caller: a warp that skips a batch leaves its masks untouched)
// DEPTH: also the per-pixel depth D = sum w * z and alpha A (depth / alpha [H,W])
// STATS: also the per-gaussian blend-weight statistics into ws (weight_stats_step / weight_stats_flush)
template <bool MARK, bool DEPTH, bool STATS = false>
__device__ __forceinline__ void render_fwd(const RecSource& rs, const int32_t* __restrict__ ranges,
                                           const float* __restrict__ background, int W, int H,
                                           int32_t* __restrict__ n_out, float* __restrict__ w_out,
                                           float* __restrict__ image, uint32_t* __restrict__ masks,
                                           const DepthSource& ds, float* __restrict__ depth,
                                           float* __restrict__ alpha, const WeightSink& ws = WeightSink{}) {
    __shared__ __align__(128) float s_rec[STAGES][BATCH * REC];
    __shared__ __align__(8) uint64_t s_full[STAGES];
    __shared__ int s_cnt[STAGES];
    __shared__ __align__(16) uint8_t s_list[CTA_WARPS][LIST_BYTES];
    __shared__ __align__(16) uint8_t s_flag[CTA_WARPS][MARK ? FLAG_BYTES : 16];  // MARK: per-record flags (fwd_walk)
    __shared__ __align__(16) float s_z[STAGES][DEPTH ? BATCH : 1];              // DEPTH: z of the staged records
    __shared__ __align__(16) uint32_t s_wacc[STAGES][STATS ? WACC_WORDS : 1];   // STATS: WeightAcc per stage

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
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
    if (lane == 0) list[LIST_DUMMY] = 0;  // made visible to the warp by the __syncwarp that ends build_lists
    const uint32_t flag_addr = smem_u32(&s_flag[warp][0]);
    if (MARK) reinterpret_cast<uint4*>(&s_flag[warp][0])[lane] = make_uint4(0u, 0u, 0u, 0u);  // likewise
    // this warp's mask words of batch 0 (the slot advances by one per batch)
    uint32_t* gm = MARK ? masks + ((size_t)(start / BATCH + tile) * MASK_WORDS_PER_SLOT + warp * GROUPS * MASK_WORDS)
                        : nullptr;

    const int nb = (total + BATCH - 1) / BATCH;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            // one arrival per lane of the refilling warp (two with DEPTH, see gather_batch)
            mbar_init(&s_full[s], DEPTH ? 64 : 32);
            s_cnt[s] = 0;
        }
        fence_mbar_init();
    }
    if (STATS)
        for (int k = tid; k < STAGES * WACC_WORDS; k += CTA_THREADS) (&s_wacc[0][0])[k] = 0u;
    __syncthreads();
    // the WHOLE calling warp fetches the records of batch b (gather_batch)
    auto load_batch = [&](int b) {
        const int s = b % STAGES;
        const int cnt = min(BATCH, total - b * BATCH);
        gather_batch<DEPTH>(rs, start + b * BATCH, cnt, &s_rec[s][0], &s_full[s], lane, &ds, &s_z[s][0]);
    };
    if (warp == 0) {
        const int pre = nb < STAGES ? nb : STAGES;
        for (int b = 0; b < pre; ++b) load_batch(b);
    }

    FwdState st;
    st.nA = pk(valid0 ? -0.0f : -1.0f, valid1 ? -0.0f : -1.0f);
    st.wl = bc(0.0f);
    st.C0 = st.C1 = st.C2 = bc(0.0f);
    st.D = bc(0.0f);
    st.last0 = st.last1 = 0;
    st.badbits = 0u;
    st.bad = false;
    const float neg_sat = -GSR_SAT_THRESH;

    for (int b = 0; b < nb; ++b) {
        const int s = b % STAGES;
        mbar_wait(&s_full[s], (uint32_t)((b / STAGES) & 1));
        const bool live0 = lo(st.nA) >= neg_sat, live1 = hi(st.nA) >= neg_sat;
        // warp-uniform: a warp whose 64 pixels are all finished only passes the stage on
        if (__any_sync(0xffffffffu, live0 || live1)) {
            const int cnt = min(BATCH, total - b * BATCH);
            const float4* rec4 = reinterpret_cast<const float4*>(&s_rec[s][0]);
            int cnts[GROUPS];
            st.bad |= build_lists<true>(rec4, cnt, lane, pm.bx0, pm.by0, list, cnts);
            const int my_cnt = group_select(cnts, lane / GROUP_LANES);
            const int iters = group_max(cnts);
            const bool small = (live0 && lo(st.nA) > -0.015625f) || (live1 && hi(st.nA) > -0.015625f);
            if (__any_sync(0xffffffffu, small)) {
                if (lane == 0) STAT(0, iters);
                fwd_walk<true, MARK, DEPTH, STATS>(rec4, list_addr, dummy_addr, my_cnt, iters, b * BATCH + 1, fpx, fpy,
                                                   st, MARK ? gm + (size_t)b * MASK_WORDS_PER_SLOT : nullptr, flag_addr,
                                                   lane, &s_z[s][0], &s_wacc[s][0]);
            } else {
                if (lane == 0) STAT(1, iters);
                fwd_walk<false, MARK, DEPTH, STATS>(rec4, list_addr, dummy_addr, my_cnt, iters, b * BATCH + 1, fpx,
                                                    fpy, st, MARK ? gm + (size_t)b * MASK_WORDS_PER_SLOT : nullptr,
                                                    flag_addr, lane, &s_z[s][0], &s_wacc[s][0]);
            }
            if (lane == 0) { STAT(5, cnts[0] + cnts[1]); STAT(6, 2 * cnt); }
#ifdef GSR_STATS
            if (lane == 0) { int sum = 0; for (int g = 0; g < GROUPS; ++g) sum += cnts[g]; STAT(4, sum); STAT(7, 1); }
#endif
        }
        if (STATS) {
            if (stage_checkout(&s_cnt[s], lane)) {  // warp-uniform: this warp left the stage last
                weight_stats_flush(&s_wacc[s][0], rs, start + b * BATCH, min(BATCH, total - b * BATCH), ws, lane);
                if (b + STAGES < nb) {
                    __syncwarp();
                    __threadfence_block();  // every lane: its share of the cleared accumulator before its arrival
                    load_batch(b + STAGES);
                }
            }
        } else if (stage_checkout(&s_cnt[s], lane) && b + STAGES < nb) {  // warp-uniform: this warp left the stage last
            load_batch(b + STAGES);
        }
    }

    // pixels flagged by the walk: recompute them exactly, one at a time, with the whole warp
    float A0 = -lo(st.nA), A1 = -hi(st.nA), wl0 = lo(st.wl), wl1 = hi(st.wl);
    float r0 = lo(st.C0), g0 = lo(st.C1), b0 = lo(st.C2), r1 = hi(st.C0), g1 = hi(st.C1), b1 = hi(st.C2);
    float D0 = lo(st.D), D1 = hi(st.D);
    // num_splats: the splat after the one that saturated the pixel, else every splat of the tile
    int n0 = (A0 > GSR_SAT_THRESH && st.last0 < total) ? st.last0 : total;
    int n1 = (A1 > GSR_SAT_THRESH && st.last1 < total) ? st.last1 : total;
    const bool bad = st.bad || (st.badbits & 0xc0000000u) != 0u;
#ifdef GSR_STATS
    if (st.bad) STAT(2, 1);
    if ((st.badbits & 0xc0000000u) != 0u) STAT(3, 1);
#endif
    uint32_t todo = __ballot_sync(0xffffffffu, bad && valid0);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int sx = __shfl_sync(0xffffffffu, px, src), sy = __shfl_sync(0xffffffffu, py, src);
        const bool two = __shfl_sync(0xffffffffu, valid1 ? 1 : 0, src) != 0;
        if (DEPTH) {
            const ExactPixelDepth e0 = render_pixel_exact_warp_depth(rs, ds, start, total, (float)sx, (float)sy, lane);
            if (lane == src) { A0 = e0.p.A; wl0 = e0.p.wl; n0 = e0.p.n; r0 = e0.p.c0; g0 = e0.p.c1; b0 = e0.p.c2; D0 = e0.d; }
            if (two) {
                const ExactPixelDepth e1 =
                    render_pixel_exact_warp_depth(rs, ds, start, total, (float)(sx + 1), (float)sy, lane);
                if (lane == src) { A1 = e1.p.A; wl1 = e1.p.wl; n1 = e1.p.n; r1 = e1.p.c0; g1 = e1.p.c1; b1 = e1.p.c2; D1 = e1.d; }
            }
            continue;
        }
        const ExactPixel e0 = render_pixel_exact_warp(rs, start, total, (float)sx, (float)sy, lane);
        if (lane == src) { A0 = e0.A; wl0 = e0.wl; n0 = e0.n; r0 = e0.c0; g0 = e0.c1; b0 = e0.c2; }
        if (two) {
            const ExactPixel e1 = render_pixel_exact_warp(rs, start, total, (float)(sx + 1), (float)sy, lane);
            if (lane == src) { A1 = e1.A; wl1 = e1.wl; n1 = e1.n; r1 = e1.c0; g1 = e1.c1; b1 = e1.c2; }
        }
    }

    const float bg0 = background[0], bg1 = background[1], bg2 = background[2];
    if (DEPTH) {  // alpha: the accumulated weight before any background; depth: no background term
        if (valid0) { depth[(size_t)py * W + px] = D0; alpha[(size_t)py * W + px] = A0; }
        if (valid1) { depth[(size_t)py * W + px + 1] = D1; alpha[(size_t)py * W + px + 1] = A1; }
    }
    auto finish = [&](bool valid, int x, float A, float wlx, int nx, float c0, float c1, float c2) {
        if (!valid) return;
        if (A < GSR_BG_THRESH) {  // src/render.cu:169-175, double arithmetic
            const double rem = 1.0 - (double)A;
            c0 = (float)fma(rem, (double)bg0, (double)c0);
            c1 = (float)fma(rem, (double)bg1, (double)c1);
            c2 = (float)fma(rem, (double)bg2, (double)c2);
        }
        const size_t pix = (size_t)py * W + x;
        n_out[pix] = nx;
        w_out[pix] = wlx;
        image[pix * 3 + 0] = c0;
        image[pix * 3 + 1] = c1;
        image[pix * 3 + 2] = c2;
    };
    finish(valid0, px, A0, wl0, n0, r0, g0, b0);
    finish(valid1, px + 1, A1, wl1, n1, r1, g1, b1);
}

template <bool MARK>
__global__ void __launch_bounds__(CTA_THREADS, GSR_FWD_MINB)
    k_render_fwd(const RecSource rs, const int32_t* __restrict__ ranges,
                 const float* __restrict__ background, int W, int H, int32_t* __restrict__ n_out,
                 float* __restrict__ w_out, float* __restrict__ image, uint32_t* __restrict__ masks) {
    render_fwd<MARK, false>(rs, ranges, background, W, H, n_out, w_out, image, masks, DepthSource{}, nullptr, nullptr);
}

#ifndef GSR_FWD_DEPTH_MINB
#define GSR_FWD_DEPTH_MINB 8
#endif
template <bool MARK>
__global__ void __launch_bounds__(CTA_THREADS, GSR_FWD_DEPTH_MINB)
    k_render_fwd_depth(const RecSource rs, const DepthSource ds, const int32_t* __restrict__ ranges,
                       const float* __restrict__ background, int W, int H, int32_t* __restrict__ n_out,
                       float* __restrict__ w_out, float* __restrict__ image, float* __restrict__ depth,
                       float* __restrict__ alpha, uint32_t* __restrict__ masks) {
    render_fwd<MARK, true>(rs, ranges, background, W, H, n_out, w_out, image, masks, ds, depth, alpha);
}

// Blend-weight statistics (weight_stats): the two forward kernels above plus the per-gaussian sums / maxima / counts.
// The group reduction keeps three more values live in the walk: at the default kernels' 9 / 8 CTAs per SM the masked
// builds spill (8-byte frame, reloaded in the walk); one CTA less (64 / 72 registers) keeps every build out of local
// memory
#ifndef GSR_FWD_STATS_MINB
#define GSR_FWD_STATS_MINB 8
#endif
#ifndef GSR_FWD_DEPTH_STATS_MINB
#define GSR_FWD_DEPTH_STATS_MINB 7
#endif
template <bool MARK>
__global__ void __launch_bounds__(CTA_THREADS, GSR_FWD_STATS_MINB)
    k_render_fwd_stats(const RecSource rs, const int32_t* __restrict__ ranges,
                       const float* __restrict__ background, int W, int H, int32_t* __restrict__ n_out,
                       float* __restrict__ w_out, float* __restrict__ image, uint32_t* __restrict__ masks,
                       const WeightSink ws) {
    render_fwd<MARK, false, true>(rs, ranges, background, W, H, n_out, w_out, image, masks, DepthSource{}, nullptr,
                                  nullptr, ws);
}
template <bool MARK>
__global__ void __launch_bounds__(CTA_THREADS, GSR_FWD_DEPTH_STATS_MINB)
    k_render_fwd_depth_stats(const RecSource rs, const DepthSource ds, const int32_t* __restrict__ ranges,
                             const float* __restrict__ background, int W, int H, int32_t* __restrict__ n_out,
                             float* __restrict__ w_out, float* __restrict__ image, float* __restrict__ depth,
                             float* __restrict__ alpha, uint32_t* __restrict__ masks, const WeightSink ws) {
    render_fwd<MARK, true, true>(rs, ranges, background, W, H, n_out, w_out, image, masks, ds, depth, alpha, ws);
}

// (float)(1.0 / (1.0 - (double)alpha)) — src/render_backward.cu:183 — without fp64: 1 - alpha is split
// exactly into hi + lo (Fast2Sum), 1/hi is refined against both its own residual and lo.  Agrees with the
// double-precision quotient rounded to float except in ~1e-7 of cases (then by one ulp), which is far below
// the reference's atomics noise; alpha <= 0.9999 so hi >= 1e-4 and nothing under/overflows.
__device__ __forceinline__ float recip_one_minus(float alpha) {
    const float hi = __fsub_rn(1.0f, alpha);
    const float lo = __fsub_rn(__fsub_rn(1.0f, hi), alpha);  // exact: (1 - hi) - alpha
    float r0;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r0) : "f"(hi));
    r0 = __fmaf_rn(r0, __fmaf_rn(-hi, r0, 1.0f), r0);        // Newton step: r0 ~ 1/hi to < 1 ulp
    const float e = __fmaf_rn(-hi, r0, 1.0f);                 // residual of r0, exact
    return __fmaf_rn(r0, __fmaf_rn(-lo, r0, e), r0);
}

// Sum 8 per-lane values across each HALF-warp (16 lanes) with 8 shuffles: every xor step halves the number
// of values a lane still carries.  On return lane L holds in v[0] its half-warp's total of value index
// 4*bit3(L) + 2*bit2(L) + bit1(L).
__device__ __forceinline__ void butterfly8_half(float* v, int lane) {
    {
        const bool up = lane & 8;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float send = up ? v[i] : v[i + 4];
            const float keep = up ? v[i + 4] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
    }
    {
        const bool up = lane & 4;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float send = up ? v[i] : v[i + 2];
            const float keep = up ? v[i + 2] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
    }
    {
        const bool up = lane & 2;
        const float send = up ? v[0] : v[1];
        const float keep = up ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
}

__device__ __forceinline__ float quarter_warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
__device__ __forceinline__ float half_warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// MASKS: the per-group splat lists come from the forward's contribution masks (exactly the records that
// contributed to the group's pixels) instead of the conservative footprint test
// DEPTH (interleaved rows only): upstream gradients on the depth and alpha maps join d_alpha through the
// same weight and r as colour, with two more back-to-front accumulators (no background term), and one more moment,
// alpha * weight * dD, is reduced and flushed into the row's slot 9 (camera-frame z)
// ABSGRAD (interleaved rows only): two more moments, sum |2c*hu - (b+b)*hv| and sum |2a*hv - (b+b)*hu| with
// the absolute value taken per pixel, before any sum; times |rdet| they are sum_p |d_u| and sum_p |d_v| (AbsGS), flushed
// into the row's slots 10 and 11.  Moments 8..11 are then gc2, z (DEPTH, else 0), |u|, |v|
template <bool MASKS, bool DEPTH, bool ABSGRAD = false>
__device__ __forceinline__ void render_bwd(const RecSource& rs,
                                           const int32_t* __restrict__ ranges, const float* __restrict__ background,
                                           int W, int H, const int32_t* __restrict__ n_in,
                                           const float* __restrict__ w_in, const float* __restrict__ grad_image,
                                           float* __restrict__ g_rgb, float* __restrict__ g_opa,
                                           float* __restrict__ g_uv, float* __restrict__ g_conic,
                                           const uint32_t* __restrict__ masks, const DepthSource& ds,
                                           const float* __restrict__ grad_depth, const float* __restrict__ grad_alpha) {
    constexpr int NG = ABSGRAD ? NGRAD + 3 : DEPTH ? NGRAD + 1 : NGRAD;  // moments per (record, batch)
    __shared__ __align__(128) float s_rec[BSTAGES][(BATCH + 1) * REC];  // + an all-zero record (alpha 0) behind each stage
    __shared__ __align__(8) uint64_t s_full[BSTAGES];
    __shared__ int s_cnt[BSTAGES];
    __shared__ float s_acc[BSTAGES][BATCH * NG];  // one moment accumulator per staged batch
    __shared__ __align__(16) uint8_t s_list[CTA_WARPS][LIST_BYTES];
    __shared__ int s_maxn;
    __shared__ __align__(16) float s_z[BSTAGES][DEPTH ? BATCH + 1 : 1];  // DEPTH: z of the staged records (+ 0)

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
    const int start = ranges[tile];
    const PixelMap pm = pixel_map(warp, lane);
    const int px = pm.px, py = pm.py;
    const bool valid0 = (px < W) && (py < H), valid1 = (px + 1 < W) && (py < H);
    const F2 fpx = pk((float)px, (float)(px + 1));
    const float fpy = (float)py;
    uint8_t* list = &s_list[warp][0];
    const uint32_t list_addr = smem_u32(list + (lane / GROUP_LANES) * BATCH);
    const uint32_t dummy_addr = smem_u32(list + LIST_DUMMY);
    if (lane == 0) list[LIST_DUMMY] = (uint8_t)BATCH;  // -> the all-zero record; visible after the CTA barriers below
    const uint32_t* gm = MASKS ? masks + ((size_t)(start / BATCH + tile) * MASK_WORDS_PER_SLOT + warp * GROUPS * MASK_WORDS)
                               : nullptr;

    int n0 = 0, n1 = 0;
    float wt0 = 0.0f, wt1 = 0.0f, da[3] = {0.f, 0.f, 0.f}, db[3] = {0.f, 0.f, 0.f};
    if (valid0) {
        const size_t pix = (size_t)py * W + px;
        n0 = n_in[pix];
        wt0 = w_in[pix];
#pragma unroll
        for (int c = 0; c < 3; ++c) da[c] = grad_image[pix * 3 + c];
    }
    if (valid1) {
        const size_t pix = (size_t)py * W + px + 1;
        n1 = n_in[pix];
        wt1 = w_in[pix];
#pragma unroll
        for (int c = 0; c < 3; ++c) db[c] = grad_image[pix * 3 + c];
    }
    F2 weight = pk(wt0, wt1);
    const F2 d0 = pk(da[0], db[0]), d1 = pk(da[1], db[1]), d2 = pk(da[2], db[2]);
    F2 dD = bc(0.0f), dA = bc(0.0f);
    if (DEPTH) {
        const size_t pix = (size_t)py * W + px;
        dD = pk(valid0 ? grad_depth[pix] : 0.0f, valid1 ? grad_depth[pix + 1] : 0.0f);
        dA = pk(valid0 ? grad_alpha[pix] : 0.0f, valid1 ? grad_alpha[pix + 1] : 0.0f);
    }
    if (tid == 0) {
        s_maxn = 0;
#pragma unroll
        for (int s = 0; s < BSTAGES; ++s) {
            mbar_init(&s_full[s], DEPTH ? 64 : 32);
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
    for (int k = tid; k < BSTAGES * BATCH * NG; k += CTA_THREADS) (&s_acc[0][0])[k] = 0.0f;
    if (tid < BSTAGES * REC) s_rec[tid / REC][BATCH * REC + tid % REC] = 0.0f;
    if (DEPTH && tid < BSTAGES) s_z[tid][BATCH] = 0.0f;
    __syncthreads();
    const int total = s_maxn;  // deepest splat any pixel of this tile consumed
    const int nb = (total + BATCH - 1) / BATCH;
    if (nb == 0) return;

    // batches are walked last -> first; pipeline slot k holds batch nb-1-k, fetched by the whole calling warp
    auto load_slot = [&](int k) {
        const int b = nb - 1 - k, s = k % BSTAGES;
        const int cnt = min(BATCH, total - b * BATCH);
        gather_batch<DEPTH>(rs, start + b * BATCH, cnt, &s_rec[s][0], &s_full[s], lane, &ds, &s_z[s][0]);
    };
    if (warp == 0) {
        const int pre = nb < BSTAGES ? nb : BSTAGES;
        for (int k = 0; k < pre; ++k) load_slot(k);
    }

    const float bg0 = background[0], bg1 = background[1], bg2 = background[2];
    F2 na0 = bc(-0.0f), na1 = bc(-0.0f), na2 = bc(-0.0f);  // -color_accum
    F2 nd = bc(-0.0f), nw = bc(-0.0f);                      // DEPTH: -acc_d, -acc_a
    bool bgi0 = false, bgi1 = false;
    const int gl = lane % GROUP_LANES;
    // after the butterfly: (16 lanes) even lanes own moments 0..7 and lane 1 the ninth; (8 lanes) every lane owns
    // one of moments 0..7 and lane 0 the ninth as well
    const int my_slot = (GROUPS == 2) ? ((gl == 1) ? 8 : (gl >> 1)) : gl;
    const bool owner = (GROUPS == 2) ? (((gl & 1) == 0) || (gl == 1)) : true;
    const uint32_t group_mask = ((GROUPS == 2) ? 0xffffu : 0xffu) << (lane & ~(GROUP_LANES - 1));


    for (int k = 0; k < nb; ++k) {
        const int b = nb - 1 - k;
        const int s = k % BSTAGES;
        const uint32_t parity = (uint32_t)((k / BSTAGES) & 1);
        const int cnt = min(BATCH, total - b * BATCH);
        mbar_wait(&s_full[s], parity);
        const float4* rec4 = reinterpret_cast<const float4*>(&s_rec[s][0]);
        float* acc = &s_acc[s][0];
        uint32_t acc_cell = smem_u32(acc) + my_slot * 4;  // this lane's moment cell of record 0
        asm volatile("" : "+r"(acc_cell));                // kept in a register: not re-derived inside the walk
        int cnts[GROUPS];
        if (MASKS)  // exactly the records that contributed to some pixel of the group
            mask_lists(gm + (size_t)b * MASK_WORDS_PER_SLOT, cnt, lane, list, cnts);
        else  // the same candidate lists the forward walked
            build_lists(rec4, cnt, lane, pm.bx0, pm.by0, list, cnts);
        const int my_cnt = group_select(cnts, lane / GROUP_LANES);
        const int iters = group_max(cnts);
        const int chunk_base1 = (b * BATCH) % CHUNK_REF + 1;  // tile_splat_idx % CHUNK of record 0 of this batch, + 1
        int base_idx = b * BATCH;
        asm volatile("" : "+r"(base_idx));  // likewise held in a register (ptxas re-derived it from k and nb per step)
#ifdef GSR_STATS
        if (lane == 0) { STAT(8, iters); STAT(10, cnts[0] + cnts[1]); STAT(13, 1); STAT(14, cnt); }
        if (lane == 0) { int sum = 0; for (int g = 0; g < GROUPS; ++g) sum += cnts[g]; STAT(15, sum); }
#endif

        // BG: handle the background term of a pixel's FIRST contribution (src/render_backward.cu:172-181).
        // -DGSR_BWD_BGSPLIT=1 compiles the walk twice and switches to the BG-less version (8 instructions per
        // iteration lighter) once every pixel of the warp is past its first contribution.  It is off by default.
        auto walk = [&](auto bg_tag) {
            constexpr bool BG = decltype(bg_tag)::value;
#pragma unroll BWD_UNROLL
        for (int step = 0; step < iters; ++step) {  // each lane group walks its own list back to front
            const int tt = my_cnt - 1 - step;
            const bool act = tt >= 0;
            const int j = (int)lds_u8(act ? list_addr + tt : dummy_addr);
            const int idx = base_idx + j;  // tile_splat_idx
            // Every rounded operation below is the one the reference's fp32 build executes for this
            // (pixel, splat) — order read off its SASS.  The weight / colour recurrences run over hundreds
            // of splats per pixel and feed cancelling differences, so "any valid fp32 order" drifts to
            // ~1e-4 of the gradient; with the same order only the summation order of the atomics differs
            // from the reference (its own run-to-run noise).
            const float4 q0 = rec4[j * 3 + 0];
            const float4 q1 = rec4[j * 3 + 1];
            const float4 q2 = rec4[j * 3 + 2];
            const float rdet = q2.x, opa = q0.w;  // 1/det (src/render_backward.cu:153), rounded once per record
            const F2 du = add2(fpx, bc(-q0.x));
            const float dv = __fsub_rn(fpy, q0.y);
            const F2 s1 = mul2(du, mul2(du, bc(q1.z)));                 // c*du*du
            const float s3 = __fmul_rn(dv, __fmul_rn(dv, q1.x));        // a*dv*dv
            const F2 s12 = fma2(bc(-dv), mul2(du, bc(q1.y)), s1);       // - (b+b)*du*dv
            const F2 mh = mul2(add2(s12, bc(s3)), bc(rdet));
            const F2 xe = mul2(mul2(mh, bc(-0.5f)), bc(LOG2E_F));
            const float g0 = lo(mh) > 0.0f ? ex2_ftz(lo(xe)) : 0.0f;
            const float g1 = hi(mh) > 0.0f ? ex2_ftz(hi(xe)) : 0.0f;
            const F2 og = mul2(pk(g0, g1), bc(opa));
            const float al0 = fminf(GSR_ALPHA_CLAMP, lo(og));  // src/render_backward.cu:167
            const float al1 = fminf(GSR_ALPHA_CLAMP, hi(og));
            // valid pixel, not beyond its saturation point (src/render_backward.cu:131), above the 1/255 skip
            // (a group past the end of its list reads the all-zero record: alpha = 0, nothing contributes)
            const bool c0 = (idx < n0) & (al0 > GSR_ALPHA_SKIP_MAX);
            const bool c1 = (idx < n1) & (al1 > GSR_ALPHA_SKIP_MAX);
            // with the forward's masks every listed record contributed to some pixel of its group: no "nobody
            // contributes" early-out is needed, a group is idle only past the end of its own list
            const uint32_t bal = MASKS ? 0xffffffffu : __ballot_sync(0xffffffffu, c0 | c1);
#ifdef GSR_STATS
            {
                const uint32_t bal = __ballot_sync(0xffffffffu, c0 | c1);  // statistics: the real contributors
                const uint32_t b0s = __ballot_sync(0xffffffffu, c0), b1s = __ballot_sync(0xffffffffu, c1);
                if (lane == 0) {
                    STAT(9, bal != 0u);
                    STAT(11, ((bal & 0xffffu) != 0u) + ((bal >> 16) != 0u));
                    STAT(12, __popc(b0s) + __popc(b1s));
                }
            }
#endif
            if (!MASKS && bal == 0u) continue;
            // a pixel that does not contribute runs the same instructions with alpha = 0: then r = 1 and the
            // weight / colour recurrences and all nine moments are left unchanged / zero
            const F2 alpha = pk(c0 ? al0 : 0.0f, c1 ? al1 : 0.0f);
            const F2 gm = pk(c0 ? g0 : 0.0f, c1 ? g1 : 0.0f);
            if (BG && ((c0 && !bgi0) || (c1 && !bgi1))) {  // src/render_backward.cu:172-181, once per pixel
                if (c0 && !bgi0) {
                    const float aw0 = __fmul_rn(lo(weight), al0);
                    const float bw = (float)(1.0 - (((double)aw0 + 1.0) - (double)lo(weight)));
                    if (bw >= GSR_BGW_MIN) {
                        na0 = pk(__fmaf_rn(bw, -bg0, lo(na0)), hi(na0));
                        na1 = pk(__fmaf_rn(bw, -bg1, lo(na1)), hi(na1));
                        na2 = pk(__fmaf_rn(bw, -bg2, lo(na2)), hi(na2));
                    }
                    bgi0 = true;
                }
                if (c1 && !bgi1) {
                    const float aw0 = __fmul_rn(hi(weight), al1);
                    const float bw = (float)(1.0 - (((double)aw0 + 1.0) - (double)hi(weight)));
                    if (bw >= GSR_BGW_MIN) {
                        na0 = pk(lo(na0), __fmaf_rn(bw, -bg0, hi(na0)));
                        na1 = pk(lo(na1), __fmaf_rn(bw, -bg1, hi(na1)));
                        na2 = pk(lo(na2), __fmaf_rn(bw, -bg2, hi(na2)));
                    }
                    bgi1 = true;
                }
            }
            const F2 r = recip_one_minus2(alpha);
            // weight recurrence with the reference's chunk-local index (SURVEY.md Q9)
            int local1 = chunk_base1 + j;  // == idx % CHUNK_REF + 1 (a batch wraps at most once)
            if (local1 > CHUNK_REF) local1 -= CHUNK_REF;
            const F2 wr = mul2(weight, r);
            weight = pk((c0 & (local1 < n0)) ? lo(wr) : lo(weight), (c1 & (local1 < n1)) ? hi(wr) : hi(weight));
            // t_c = weight*col_c - r*acc_c ; d_alpha = sum_c dC_c * t_c
            const F2 t0 = fma2(weight, bc(q2.y), mul2(r, na0));
            const F2 t1 = fma2(weight, bc(q2.z), mul2(r, na1));
            const F2 t2 = fma2(weight, bc(q2.w), mul2(r, na2));
            F2 galpha = fma2(d2, t2, fma2(d1, t1, fma2(d0, t0, bc(0.0f))));
            float zj = 0.0f;
            if (DEPTH) {  // d_alpha += (z*weight - acc_d*r)*dD + (weight - acc_a*r)*dA
                zj = s_z[s][j];
                const F2 td = fma2(weight, bc(zj), mul2(r, nd));
                const F2 ta = fma2(r, nw, weight);
                galpha = fma2(dA, ta, fma2(dD, td, galpha));
            }
            // acc_c += weight * (alpha * col_c), kept negated
            na0 = fma2(weight, mul2(alpha, bc(-q2.y)), na0);
            na1 = fma2(weight, mul2(alpha, bc(-q2.z)), na1);
            na2 = fma2(weight, mul2(alpha, bc(-q2.w)), na2);
            if (DEPTH) {  // acc_d += weight * (alpha * z), acc_a += weight * alpha, kept negated
                nd = fma2(weight, mul2(alpha, bc(-zj)), nd);
                nw = fma2(weight, mul2(alpha, bc(-1.0f)), nw);
            }
            // Only nine per-pixel MOMENTS are reduced; the uv / conic gradient formulas
            // (src/render_backward.cu:216-229) are linear in them and are finished once per
            // (gaussian, tile) pair after the reduction, in the flush below:
            //   S0..2 = alpha*weight*dC_c          -> d_rgb_c   = SH_0 * S_c
            //   S3    = g * d_alpha                 -> d_opacity
            //   S4,S5 = gmh*du, gmh*dv              -> d_u, d_v
            //   S6..8 = gmh*du*du, gmh*du*dv, gmh*dv*dv -> d_conic
            const F2 aw = mul2(alpha, weight);
            // reference: (float)(-0.5 * g * gprob) in double; the double product of two floats is exact,
            // so one fp32 rounding of it is the same value
            const F2 gmh = mul2(mul2(gm, bc(-0.5f)), mul2(bc(opa), galpha));
            const F2 hu = mul2(gmh, du), hv = mul2(gmh, bc(dv));
            const F2 m0 = mul2(d0, aw), m1 = mul2(d1, aw), m2 = mul2(d2, aw), m3 = mul2(galpha, gm);
            const F2 m6 = mul2(hu, du), m7 = mul2(hu, bc(dv)), m8 = mul2(hv, bc(dv));
            float g8[8];
            g8[0] = lo(m0) + hi(m0);
            g8[1] = lo(m1) + hi(m1);
            g8[2] = lo(m2) + hi(m2);
            g8[3] = lo(m3) + hi(m3);
            g8[4] = lo(hu) + hi(hu);
            g8[5] = lo(hv) + hi(hv);
            g8[6] = lo(m6) + hi(m6);
            g8[7] = lo(m7) + hi(m7);
            float gc2 = lo(m8) + hi(m8);
            float gz = 0.0f;  // DEPTH: S9 = alpha*weight*dD -> d_z
            if (DEPTH) {
                const F2 mz = mul2(dD, aw);
                gz = lo(mz) + hi(mz);
            }
            // ABSGRAD: S10, S11 = |2c*hu - (b+b)*hv|, |2a*hv - (b+b)*hu| per pixel (d_u = -rdet * eu, d_v = -rdet * ev)
            float gau = 0.0f, gav = 0.0f;
            if (ABSGRAD) {
                const F2 eu = fma2(bc(q1.z + q1.z), hu, mul2(bc(-q1.y), hv));
                const F2 ev = fma2(bc(q1.x + q1.x), hv, mul2(bc(-q1.y), hu));
                gau = fabsf(lo(eu)) + fabsf(hi(eu));
                gav = fabsf(lo(ev)) + fabsf(hi(ev));
            }
            const bool group_any = MASKS ? act : ((bal & group_mask) != 0u);
            if (GROUPS == 2) {
                butterfly8_half(g8, lane);
                gc2 = half_warp_sum(gc2);
                if (DEPTH) gz = half_warp_sum(gz);
                const float mine = (gl == 1) ? gc2 : g8[0];
                if (group_any & owner) atomicAdd(&acc[j * NG + my_slot], mine);
                if (DEPTH && group_any && gl == 0) atomicAdd(&acc[j * NG + NGRAD], gz);
                if (ABSGRAD) {
                    gau = half_warp_sum(gau);
                    gav = half_warp_sum(gav);
                    if (group_any && gl == 2) atomicAdd(&acc[j * NG + NGRAD + 1], gau);
                    if (group_any && gl == 3) atomicAdd(&acc[j * NG + NGRAD + 2], gav);
                }
            } else if (ABSGRAD) {
                // moments 8..11 reduced together: lane gl < 4 of the group ends with moment 8 + gl and adds it with
                // the same atomic instruction as the others' share of moments 0..7
                butterfly8_quarter(g8, lane);
                float t4[4] = {gc2, gz, gau, gav};
                butterfly4_quarter_low(t4, lane);
                if (group_any) {
                    float* cell = reinterpret_cast<float*>(__cvta_shared_to_generic(acc_cell + j * (NG * 4)));
                    atomicAdd(cell, g8[0]);
                    if (gl < 4) atomicAdd(cell + 8, t4[0]);
                }
            } else {
                butterfly8_quarter(g8, lane);
                gc2 = quarter_warp_sum(gc2);
                if (DEPTH) gz = quarter_warp_sum(gz);
                if (group_any) {
                    float* cell = reinterpret_cast<float*>(__cvta_shared_to_generic(acc_cell + j * (NG * 4)));
                    atomicAdd(cell, g8[0]);
                    if (gl == 0) atomicAdd(cell + 8, gc2);
                    if (DEPTH && gl == 1) atomicAdd(cell + 8, gz);  // lane 1's cell + 8 is moment 9
                }
            }
        }
        };
#if GSR_BWD_BGSPLIT
        const bool bg_pending = (!bgi0 && n0 > 0) || (!bgi1 && n1 > 0);
        if (__any_sync(0xffffffffu, bg_pending)) walk(std::true_type{});
        else walk(std::false_type{});
#else
        walk(std::true_type{});
#endif
        // The last warp to finish this batch finishes the gradient formulas from the nine moments of each
        // pair (one atomic per (pair, component)), clears the accumulator and recycles the stage.
        if (stage_checkout(&s_cnt[s], lane)) {
            int gids[BATCH / 32];  // all loads first: one global-memory latency per batch, not four
#pragma unroll
            for (int i = 0; i < BATCH / 32; ++i) {
                const int r = lane + 32 * i;
                gids[i] = (r >= cnt) ? 0 : (int)source_id(rs, start + b * BATCH + r);
            }
#pragma unroll
            for (int i = 0; i < BATCH / 32; ++i) {
                const int r = lane + 32 * i;
                if (r >= cnt) break;
                float S[NG];
                bool any = false;
#pragma unroll
                for (int q = 0; q < NG; ++q) {
                    S[q] = acc[r * NG + q];
                    any |= (S[q] != 0.0f);
                }
                if (any) {
#pragma unroll
                    for (int q = 0; q < NG; ++q) acc[r * NG + q] = 0.0f;
                    const float4 q1 = rec4[r * 3 + 1];
                    const float a = q1.x, bh = 0.5f * q1.y, c = q1.z, rdet = rec4[r * 3 + 2].x;
                    const int gid = gids[i];
                    // d_u = -(2c du - 2b dv) rdet gmh ; d_v = -(2a dv - 2b du) rdet gmh   (render_backward.cu:216-219)
                    const float gu = -rdet * (2.0f * c * S[4] - 2.0f * bh * S[5]);
                    const float gv = -rdet * (2.0f * a * S[5] - 2.0f * bh * S[4]);
                    // common_frac summed over pixels (render_backward.cu:221-223)
                    const float cf = (a * S[8] - 2.0f * bh * S[7] + c * S[6]) * rdet * rdet;
                    const float gc0 = -c * cf + S[8] * rdet, gc1 = bh * cf - S[7] * rdet, gc2 = -a * cf + S[6] * rdet;
                    if (DEPTH || ABSGRAD || g_opa == nullptr) {
                        // interleaved gradient rows [gaussian][12] = rgb3 opa | uv2 conic0 conic1 | conic2 pad3: the
                        // nine sums of a pair land in two adjacent 32-byte sectors through two 16-byte vector
                        // reductions + one scalar (planar arrays: nine scalar reductions into four arrays).
                        // DEPTH: conic2 z pad2, the last two through one 8-byte vector reduction.
                        // ABSGRAD: conic2 z|0 |u| |v|, the whole tail through a third 16-byte vector reduction
                        float* row = g_rgb + (size_t)gid * GRAD_ROW;
                        red_add_v4(row, GSR_SH0 * S[0], GSR_SH0 * S[1], GSR_SH0 * S[2], S[3]);
                        red_add_v4(row + 4, gu, gv, gc0, gc1);
                        if (ABSGRAD)
                            red_add_v4(row + 8, gc2, DEPTH ? S[NGRAD] : 0.0f, fabsf(rdet) * S[NGRAD + 1],
                                       fabsf(rdet) * S[NGRAD + 2]);
                        else if (DEPTH)
                            red_add_v2(row + 8, gc2, S[NG - 1]);
                        else
                            atomicAdd(row + 8, gc2);
                    } else {
                        atomicAdd(g_rgb + (size_t)gid * 3 + 0, GSR_SH0 * S[0]);
                        atomicAdd(g_rgb + (size_t)gid * 3 + 1, GSR_SH0 * S[1]);
                        atomicAdd(g_rgb + (size_t)gid * 3 + 2, GSR_SH0 * S[2]);
                        atomicAdd(g_opa + gid, S[3]);
                        atomicAdd(g_uv + (size_t)gid * 2 + 0, gu);
                        atomicAdd(g_uv + (size_t)gid * 2 + 1, gv);
                        atomicAdd(g_conic + (size_t)gid * 3 + 0, gc0);
                        atomicAdd(g_conic + (size_t)gid * 3 + 1, gc1);
                        atomicAdd(g_conic + (size_t)gid * 3 + 2, gc2);
                    }
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

template <bool MASKS>
__global__ void __launch_bounds__(CTA_THREADS, GSR_BWD_MINB)
    k_render_bwd(const RecSource rs,
                 const int32_t* __restrict__ ranges, const float* __restrict__ background, int W, int H,
                 const int32_t* __restrict__ n_in, const float* __restrict__ w_in,
                 const float* __restrict__ grad_image, float* __restrict__ g_rgb,
                 float* __restrict__ g_opa, float* __restrict__ g_uv, float* __restrict__ g_conic,
                 const uint32_t* __restrict__ masks) {
    render_bwd<MASKS, false>(rs, ranges, background, W, H, n_in, w_in, grad_image, g_rgb, g_opa, g_uv, g_conic, masks,
                             DepthSource{}, nullptr, nullptr);
}

#ifndef GSR_BWD_DEPTH_MINB
// the two more per-pixel upstream gradients and accumulators do not fit the default build's 64 registers: at 72 (7 CTAs)
// the masked walk reloads a spilled register every iteration, at 80 (6 CTAs) once per batch; at 5 CTAs (88-89
// registers) neither variant keeps anything in local memory
#define GSR_BWD_DEPTH_MINB 5
#endif
template <bool MASKS>
__global__ void __launch_bounds__(CTA_THREADS, GSR_BWD_DEPTH_MINB)
    k_render_bwd_depth(const RecSource rs, const DepthSource ds, const int32_t* __restrict__ ranges,
                       const float* __restrict__ background, int W, int H, const int32_t* __restrict__ n_in,
                       const float* __restrict__ w_in, const float* __restrict__ grad_image,
                       const float* __restrict__ grad_depth, const float* __restrict__ grad_alpha,
                       float* __restrict__ grad_rows, const uint32_t* __restrict__ masks) {
    render_bwd<MASKS, true>(rs, ranges, background, W, H, n_in, w_in, grad_image, grad_rows, nullptr, nullptr, nullptr,
                            masks, ds, grad_depth, grad_alpha);
}

// Absolute uv gradients (GSR_MODE_ABSGRAD), colour only or with depth/alpha (DEPTH).  The two more moments are
// transient per step (no per-pixel state persists), so the masked colour-only kernel keeps the default 8 CTAs per SM
// with no local memory, and the depth ones the depth kernel's 5; s_acc grows to 12 floats per record (27.8 KB of shared
// memory: 8 CTAs still fit).  The colour-only kernel without masks also carries the candidate-list build: at 8 CTAs it
// spills (32-byte frame, reloaded in the walk), at 7 (72 registers) still 8 bytes; at 6 (78 registers) nothing
#ifndef GSR_BWD_ABS_MINB
#define GSR_BWD_ABS_MINB 8
#endif
#ifndef GSR_BWD_ABS_NOMASK_MINB
#define GSR_BWD_ABS_NOMASK_MINB 6
#endif
#ifndef GSR_BWD_DEPTH_ABS_MINB
#define GSR_BWD_DEPTH_ABS_MINB 5
#endif
template <bool MASKS, bool DEPTH>
__global__ void __launch_bounds__(CTA_THREADS, DEPTH   ? GSR_BWD_DEPTH_ABS_MINB
                                               : MASKS ? GSR_BWD_ABS_MINB
                                                       : GSR_BWD_ABS_NOMASK_MINB)
    k_render_bwd_abs(const RecSource rs, const DepthSource ds, const int32_t* __restrict__ ranges,
                     const float* __restrict__ background, int W, int H, const int32_t* __restrict__ n_in,
                     const float* __restrict__ w_in, const float* __restrict__ grad_image,
                     const float* __restrict__ grad_depth, const float* __restrict__ grad_alpha,
                     float* __restrict__ grad_rows, const uint32_t* __restrict__ masks) {
    render_bwd<MASKS, DEPTH, true>(rs, ranges, background, W, H, n_in, w_in, grad_image, grad_rows, nullptr, nullptr,
                                   nullptr, masks, ds, grad_depth, grad_alpha);
}

}  // namespace gsr

using namespace gsr;

// the sort-key depth field of the pair list (or the per-gaussian depth keys, sorted id array): see DepthSource
static bool make_depth_source(const uint64_t* keys_sorted, int id_bits, const uint32_t* depth_key,
                              uint32_t depth_base, int depth_bits, DepthSource& ds) {
    if (depth_bits < 1 || depth_bits > 32) return false;
    if (depth_base == 0u && depth_bits != 32) return false;  // depth_key()'s transform uses all 32 bits
    if (keys_sorted == nullptr && depth_key == nullptr) return false;
    if (keys_sorted != nullptr && (id_bits <= 0 || id_bits + depth_bits > 64)) return false;
    ds.zkey = depth_key;
    ds.depth_base = depth_base;
    ds.depth_mask = depth_bits == 32 ? ~0u : ((1u << depth_bits) - 1u);
    ds.id_bits = keys_sorted != nullptr ? id_bits : 0;
    return true;
}

// ds != nullptr: the depth/alpha kernels; ws != nullptr: the blend-weight statistics kernels
static int launch_forward(const RecSource& src, const DepthSource* ds, const int32_t* ranges, const float* background,
                          int H, int W, int32_t* n_out, float* w_out, float* image, float* depth, float* alpha,
                          uint32_t* masks, const WeightSink* ws, void* stream) {
    if (H <= 0 || W <= 0) return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE), block(CTA_THREADS);
    cudaStream_t st = (cudaStream_t)stream;
    if (ws != nullptr) {
        const DepthSource d = ds != nullptr ? *ds : DepthSource{};
        if (ds != nullptr && masks != nullptr)
            k_render_fwd_depth_stats<true><<<grid, block, 0, st>>>(src, d, ranges, background, W, H, n_out, w_out,
                                                                   image, depth, alpha, masks, *ws);
        else if (ds != nullptr)
            k_render_fwd_depth_stats<false><<<grid, block, 0, st>>>(src, d, ranges, background, W, H, n_out, w_out,
                                                                    image, depth, alpha, nullptr, *ws);
        else if (masks != nullptr)
            k_render_fwd_stats<true><<<grid, block, 0, st>>>(src, ranges, background, W, H, n_out, w_out, image, masks,
                                                             *ws);
        else
            k_render_fwd_stats<false><<<grid, block, 0, st>>>(src, ranges, background, W, H, n_out, w_out, image,
                                                              nullptr, *ws);
    } else if (ds != nullptr) {
        if (masks != nullptr)
            k_render_fwd_depth<true><<<grid, block, 0, st>>>(src, *ds, ranges, background, W, H, n_out, w_out, image,
                                                             depth, alpha, masks);
        else
            k_render_fwd_depth<false><<<grid, block, 0, st>>>(src, *ds, ranges, background, W, H, n_out, w_out, image,
                                                              depth, alpha, nullptr);
    } else if (masks != nullptr) {
        k_render_fwd<true><<<grid, block, 0, st>>>(src, ranges, background, W, H, n_out, w_out, image, masks);
    } else {
        k_render_fwd<false><<<grid, block, 0, st>>>(src, ranges, background, W, H, n_out, w_out, image, nullptr);
    }
    return (int)cudaGetLastError();
}

// ds != nullptr: the depth/alpha kernels; absgrad: the absolute-uv-gradient kernels (both write interleaved rows,
// passed as g_rgb)
static int launch_backward(const RecSource& src, const DepthSource* ds, bool absgrad, const int32_t* ranges, const float* background, int H, int W, const int32_t* n_in,
                           const float* w_in, const float* grad_image, const float* grad_depth,
                           const float* grad_alpha, float* g_rgb, float* g_opa, float* g_uv, float* g_conic,
                           const uint32_t* masks, void* stream) {
    if (H <= 0 || W <= 0) return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE), block(CTA_THREADS);
    cudaStream_t st = (cudaStream_t)stream;
    if (absgrad) {
        const DepthSource d = ds != nullptr ? *ds : DepthSource{};
        if (ds != nullptr && masks != nullptr)
            k_render_bwd_abs<true, true><<<grid, block, 0, st>>>(src, d, ranges, background, W, H, n_in, w_in,
                                                                 grad_image, grad_depth, grad_alpha, g_rgb, masks);
        else if (ds != nullptr)
            k_render_bwd_abs<false, true><<<grid, block, 0, st>>>(src, d, ranges, background, W, H, n_in, w_in,
                                                                  grad_image, grad_depth, grad_alpha, g_rgb, nullptr);
        else if (masks != nullptr)
            k_render_bwd_abs<true, false><<<grid, block, 0, st>>>(src, d, ranges, background, W, H, n_in, w_in,
                                                                  grad_image, nullptr, nullptr, g_rgb, masks);
        else
            k_render_bwd_abs<false, false><<<grid, block, 0, st>>>(src, d, ranges, background, W, H, n_in, w_in,
                                                                   grad_image, nullptr, nullptr, g_rgb, nullptr);
    } else if (ds != nullptr) {
        if (masks != nullptr)
            k_render_bwd_depth<true><<<grid, block, 0, st>>>(src, *ds, ranges, background, W, H, n_in, w_in,
                                                             grad_image, grad_depth, grad_alpha, g_rgb, masks);
        else
            k_render_bwd_depth<false><<<grid, block, 0, st>>>(src, *ds, ranges, background, W, H, n_in, w_in,
                                                              grad_image, grad_depth, grad_alpha, g_rgb, nullptr);
    } else if (masks != nullptr) {
        k_render_bwd<true><<<grid, block, 0, st>>>(src, ranges, background, W, H, n_in, w_in, grad_image, g_rgb, g_opa,
                                                   g_uv, g_conic, masks);
    } else {
        k_render_bwd<false><<<grid, block, 0, st>>>(src, ranges, background, W, H, n_in, w_in, grad_image, g_rgb, g_opa,
                                                    g_uv, g_conic, nullptr);
    }
    return (int)cudaGetLastError();
}

extern "C" {

size_t gsr_contribution_mask_words(int64_t P, int H, int W) {
    if (P < 0 || H <= 0 || W <= 0) return 0;
    const int64_t n_tiles = (int64_t)((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    return (size_t)(P / BATCH + n_tiles + 1) * MASK_WORDS_PER_SLOT;
}

int gsr_render_forward_gather(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                              const int32_t* ids_sorted, const uint32_t* depth_key, uint32_t depth_base, int depth_bits,
                              const int32_t* ranges, const float* background, int H, int W, int32_t* n_out,
                              float* w_out, float* image, float* depth, float* alpha, uint32_t* contribution_masks,
                              void* stream) {
    if ((keys_sorted == nullptr) == (ids_sorted == nullptr)) return GSR_ERR_BAD_ARG;  // exactly one id source
    if ((depth == nullptr) != (alpha == nullptr)) return GSR_ERR_BAD_ARG;
    DepthSource ds;
    if (depth != nullptr && !make_depth_source(keys_sorted, id_bits, depth_key, depth_base, depth_bits, ds))
        return GSR_ERR_BAD_ARG;
    return launch_forward(make_source(gaussian_records, keys_sorted, ids_sorted, id_bits),
                          depth != nullptr ? &ds : nullptr, ranges, background, H, W, n_out, w_out, image, depth, alpha,
                          contribution_masks, nullptr, stream);
}

int gsr_render_forward_gather_stats(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                                    const int32_t* ids_sorted, const uint32_t* depth_key, uint32_t depth_base,
                                    int depth_bits, const int32_t* ranges, const float* background, int H, int W,
                                    int32_t* n_out, float* w_out, float* image, float* depth, float* alpha,
                                    uint32_t* contribution_masks, float* weight_sum, float* weight_max,
                                    int32_t* pixel_count, const uint64_t* pair_total, int64_t pair_capacity,
                                    void* stream) {
    const int given = (weight_sum != nullptr) + (weight_max != nullptr) + (pixel_count != nullptr);
    if (given == 0)
        return gsr_render_forward_gather(gaussian_records, keys_sorted, id_bits, ids_sorted, depth_key, depth_base,
                                         depth_bits, ranges, background, H, W, n_out, w_out, image, depth, alpha,
                                         contribution_masks, stream);
    if (given != 3) return GSR_ERR_BAD_ARG;
    if (pair_total != nullptr && (pair_capacity < 0 || pair_capacity > 0xffffffffll)) return GSR_ERR_BAD_ARG;
    if ((keys_sorted == nullptr) == (ids_sorted == nullptr)) return GSR_ERR_BAD_ARG;  // exactly one id source
    if ((depth == nullptr) != (alpha == nullptr)) return GSR_ERR_BAD_ARG;
    DepthSource ds;
    if (depth != nullptr && !make_depth_source(keys_sorted, id_bits, depth_key, depth_base, depth_bits, ds))
        return GSR_ERR_BAD_ARG;
    WeightSink ws;
    ws.sum = weight_sum;
    ws.max = reinterpret_cast<uint32_t*>(weight_max);
    ws.count = reinterpret_cast<uint32_t*>(pixel_count);
    ws.pair_total = pair_total;
    ws.capacity = pair_total != nullptr ? (uint32_t)pair_capacity : 0u;
    return launch_forward(make_source(gaussian_records, keys_sorted, ids_sorted, id_bits),
                          depth != nullptr ? &ds : nullptr, ranges, background, H, W, n_out, w_out, image, depth, alpha,
                          contribution_masks, &ws, stream);
}

int gsr_render_backward_gather(int mode, const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                               const int32_t* ids_sorted, const uint32_t* depth_key, uint32_t depth_base,
                               int depth_bits, const int32_t* ranges, const float* background, int H, int W,
                               const int32_t* n_in, const float* w_in, const float* grad_image,
                               const float* grad_depth, const float* grad_alpha, float* g_rgb, float* g_opa,
                               float* g_uv, float* g_conic, float* grad_rows, const uint32_t* contribution_masks,
                               void* stream) {
    // the other stages' bits are accepted and ignored: depth/alpha is selected by the maps' gradients
    if ((mode & ~(GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D)) != 0)
        return GSR_ERR_BAD_ARG;
    const bool absgrad = (mode & GSR_MODE_ABSGRAD) != 0;
    if (absgrad && grad_rows == nullptr) return GSR_ERR_BAD_ARG;  // slots 10-11 exist only in the interleaved rows
    if ((keys_sorted == nullptr) == (ids_sorted == nullptr)) return GSR_ERR_BAD_ARG;
    if (grad_image == nullptr || (grad_depth == nullptr) != (grad_alpha == nullptr)) return GSR_ERR_BAD_ARG;
    DepthSource ds;
    if (grad_depth != nullptr &&
        (grad_rows == nullptr || !make_depth_source(keys_sorted, id_bits, depth_key, depth_base, depth_bits, ds)))
        return GSR_ERR_BAD_ARG;
    if (grad_rows != nullptr) {  // interleaved rows: the kernel sees them as g_rgb with the other three NULL
        if ((reinterpret_cast<uintptr_t>(grad_rows) & 15u) != 0) return GSR_ERR_BAD_ARG;
        g_rgb = grad_rows;
        g_opa = g_uv = g_conic = nullptr;
    } else if (g_rgb == nullptr || g_opa == nullptr || g_uv == nullptr || g_conic == nullptr) {
        return GSR_ERR_BAD_ARG;
    }
    return launch_backward(make_source(gaussian_records, keys_sorted, ids_sorted, id_bits),
                           grad_depth != nullptr ? &ds : nullptr, absgrad, ranges, background, H, W, n_in, w_in,
                           grad_image, grad_depth, grad_alpha, g_rgb, g_opa, g_uv, g_conic, contribution_masks, stream);
}

const char* gsr_version(void) { return "gsr_b200 0.1 sm_90a"; }

#ifdef GSR_STATS
int gsr_debug_stats(unsigned long long* out, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, g_stats, sizeof(unsigned long long) * 16);
    if (reset) {
        unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(g_stats, z, sizeof(z));
    }
    return 0;
}
#endif

}  // extern "C"
