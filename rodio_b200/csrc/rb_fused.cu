// rb_fused.cu — the fused resample -> channel-map -> effects -> mix kernel (fast path).
//
// Shape covered (every stream of the batch must have the same adapter-kind sequence; parameters are
// per stream):   [convert] [amplify]*  [uniform]?  [amplify]* [biquad]? [amplify]*   -> mixer sum
// i.e. BASELINE cfg2 (plain mixer of sources) and cfg3 (resample -> low_pass -> amplify -> mix), in any
// channel layout.  Everything else is served by the general per-adapter kernels (rb_kernels.cu).
//
// Work decomposition (H100: 132 SMs, 4 sub-partitions each, 1 warp-instruction / cycle / sub-partition):
//   * a CTA owns G consecutive streams ("rows", insertion order) and walks the mixer timeline in tiles
//     of TT samples; G is chosen so that the grid is one balanced wave over the SMs.
//   * per tile three stages run CONCURRENTLY on three different tiles (software pipeline over a ring of
//     three shared-memory tile buffers, one __syncthreads per tile):
//       A  (all "parallel" warps)  tile k   : input taps -> pre-gains -> linear interpolation + channel map
//                                             -> gains  => x[row][t] in shared memory; loads are coalesced
//                                             along time and every input sample is fetched from HBM once.
//       B  (recurrence warps)      tile k-1 : Direct-Form-I biquad, one lane per (row, channel) chain,
//                                             strictly the reference's f32 operation order (bit-exact);
//                                             state lives in registers across tiles.
//       C  (parallel warps)        tile k-2 : post-gains and the ordered sum over the CTA's rows
//                                             -> one partial-mix row per CTA in HBM.
//     The recurrence is a 12-cycle dependent chain per sample (FMUL -> FADD -> FADD): it is the critical
//     path at modest batch sizes, so stage B owns its warps and never waits for loads.
//   * a second tiny kernel adds the per-CTA partial rows in CTA order (deterministic).  With one CTA the
//     result equals the reference's strictly sequential sum bit for bit.
//
// Without a biquad the kernel degenerates to stage A + C in registers (no shared memory, no barrier).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "rb_dsp.cuh"
#include "rb_fused.h"
#include "rb_lanes.h"
#include "rb_fused_rows.h"   // FusedRow, ROW_*, TT, MAX_GAINS, parse_row, fused_lanes_hook (host-visible: also run by the CPU suite)

using namespace rbd;

namespace {

constexpr int ROW_STRIDE = TT + 4; // words; (TT+4)/4 odd -> LDS.128 by 8 lanes hits 8 distinct bank groups
constexpr int HOT_PAD = 4;          // k_fused_hot: tile position 0 sits at word 4 of its row; words 2,3 hold x[-2], x[-1]
constexpr int MAX_G = 32;          // rows per CTA
constexpr int NBUF = 3;

struct FusedArgs {
    const FusedRow* rows;
    uint32_t n_rows;
    uint32_t rows_per_cta;
    uint32_t c_mix;                // mixer channels
    uint32_t n_pre, n_mid, n_post;
    uint32_t has_biquad;
    float* partial;                // [n_ctas][mix_len]
    uint64_t mix_len;
    uint32_t direct;               // single CTA: `partial` is the mixer output itself, cover the whole timeline
    uint32_t chain;                // RB_MIX_EXACT_ORDER on k_fused_hot: CTA c starts every tile's sum from the running sum CTA c - 1
                                   // left for that tile -- the reference's sequential order over ALL streams (src/mixer.rs:185-198)
    float* out;                    // chain: the last CTA's row is the mixer output
    uint32_t* flags;               // chain: one word, the ticket counter (never reset: tickets of render e start at e * n_ctas)
    uint32_t epoch;                // chain: render number, part of every tag
    uint32_t win_stride;           // k_fused_hot: floats per row window (WSTRIDE or WSTRIDE_NARROW)
};

// ---- per (row, tile) index state -------------------------------------------------------------------
struct RowTile {
    uint32_t lo, hi;       // active tile positions [lo, hi)
    uint32_t r0;           // ROW_LERP: (n0 * from) mod to at frame n0
    uint32_t j0;           // channel of the first active sample (o0 % c_mix)
    uint64_t i0;           // ROW_LERP: left input frame of frame n0 ; ROW_PASS: n0
    uint64_t o0;           // row-local output sample index at tile position `lo`
};

__device__ __forceinline__ float apply_gains(float v, const float* g, uint32_t n) {
#pragma unroll
    for (int k = 0; k < MAX_GAINS; k++)
        if (k < (int)n) v = mul(v, g[k]);
    return v;
}

template <bool NOGAIN>
__device__ __forceinline__ float gains(float v, const float* g, uint32_t n) {
    return NOGAIN ? v : apply_gains(v, g, n);
}

template <bool F32>
__device__ __forceinline__ float load_in(const void* in, uint32_t fmt, uint64_t idx) {
    if (F32) return __ldg((const float*)in + idx);
    return load_as_f32(in, fmt, idx);
}

// (b - a) * num / den with the reference's rounding sequence, the division done as an exact
// reciprocal refinement: q0 = RN(m * rcp); r = m - q0 * den (exact, FMA); q = RN(q0 + r * rcp) == RN(m / den)
// (Markstein).  Outside the guarded range (zeros keep their sign, denormals, huge values) fall back to the
// IEEE division.  Verified exhaustively against `/` for every den <= 4000 and the common rate pairs.
__device__ __forceinline__ float lerp_rcp(float first, float second, float num_f, float den_f, float rcp_den) {
    float m = mul(sub(second, first), num_f);
    float am = fabsf(m);
    float q0 = mul(m, rcp_den);
    float r = __fmaf_rn(-q0, den_f, m);
    float q = __fmaf_rn(r, rcp_den, q0);
    q = (am == 0.0f) ? m : q;                                   // (+-0) / den keeps its sign
    const bool rare = !(am <= 1e30f) || (am < 1e-30f && am != 0.0f);          // denormal / huge / NaN operand
    if (__any_sync(__activemask(), rare)) q = rare ? divf(m, den_f) : q;      // warp-uniform branch, never taken on audio
    return add(first, q);
}

// Generic (any segment / partial frame / chunk boundary) sample of the row at local output index o.
template <bool F32>
__device__ __noinline__ float row_sample_generic(const FusedRow& r, uint32_t c_mix, uint32_t n_pre, uint32_t n_mid,
                                                 uint64_t o) {
    if (!r.has_uniform) return apply_gains(apply_gains(load_in<F32>(r.in, r.fmt, o), r.pre, n_pre), r.mid, n_mid);
    UniformTap t = uniform_tap(r.uni, r.c_in, c_mix, o);
    float v = 0.0f;
    if (t.kind != 0) {
        float x0 = apply_gains(load_in<F32>(r.in, r.fmt, t.i0), r.pre, n_pre);
        v = x0;
        if (t.kind == 2) {
            float x1 = apply_gains(load_in<F32>(r.in, r.fmt, t.i0 + r.c_in), r.pre, n_pre);
            v = lerp_f(x0, x1, __uint2float_rn(t.num), r.den_f);
        }
    }
    return apply_gains(v, r.mid, n_mid);
}

__device__ __forceinline__ void row_tile_setup(const FusedRow& r, uint32_t c_mix, uint64_t m0, RowTile& rt) {
    uint64_t s = r.mix_start, e = r.mix_start + r.out_len;
    uint64_t lo = m0 > s ? m0 : s, hi = (m0 + TT) < e ? (m0 + TT) : e;
    rt.lo = rt.hi = 0, rt.r0 = 0, rt.j0 = 0, rt.i0 = 0, rt.o0 = 0;
    if (lo >= hi) return;
    rt.lo = (uint32_t)(lo - m0), rt.hi = (uint32_t)(hi - m0);
    rt.o0 = lo - s;
    uint64_t n0 = rt.o0 / c_mix;
    rt.j0 = (uint32_t)(rt.o0 - n0 * c_mix);
    if (r.mode == ROW_LERP) {
        uint64_t prod = n0 * (uint64_t)r.uni.from;
        rt.i0 = prod / r.uni.to;
        rt.r0 = (uint32_t)(prod - rt.i0 * r.uni.to);
    } else {
        rt.i0 = n0;
    }
}

// Stage A, hot case: mono source, mono mixer, linear interpolation (BASELINE cfg3).  One batch of 8 output
// frames per lane covers the tile; indices are 32-bit offsets from the tile's first input frame.
template <bool F32, bool NOGAIN>
__device__ __forceinline__ void stage_a_mono_lerp(const FusedRow& r, const RowTile& rt, uint32_t n_pre, uint32_t n_mid,
                                                  uint32_t lane, float* __restrict__ row) {
    constexpr int U = TT / 32;   // output frames per lane per tile
    constexpr int H = 4;         // frames per half-batch: 2*H independent loads in flight per lane
    const uint32_t n = rt.hi - rt.lo;
    const uint32_t to = r.uni.to, q32 = r.q32, r32 = r.r32, fmt = r.fmt;
    const float den_f = r.den_f, rcp_den = r.rcp_den;
    const uint64_t remain = r.uni.tail.L - 1 - rt.i0;              // frames to the right of i0
    const uint32_t lim = remain > 0x7fffffffull ? 0x7fffffffu : (uint32_t)remain;   // interpolate iff di < lim
    const float* __restrict__ base_f = (const float*)r.in + rt.i0;
    const float* pre = r.pre;   // shared memory (warp-broadcast reads); only touched when gains exist
    const float* mid = r.mid;
    uint32_t prod = rt.r0 + lane * r.uni.from;
    uint32_t di = prod / to;
    uint32_t num = prod - di * to;
    float* __restrict__ out = row + rt.lo + lane;
    // last left index this lane will touch in the tile: di + (U-1) * (32*from/to) rounded up
    const bool interior = F32 && n == (uint32_t)TT && (di + (uint32_t)(U - 1) * (q32 + 1) + 1) < lim;
    if (interior) {
        // every position active, every right neighbour exists -> no predicates at all
#pragma unroll 1
        for (int h = 0; h < U; h += H) {
            uint32_t dis[H];
            float nf[H], x0[H], x1[H];
#pragma unroll
            for (int u = 0; u < H; u++) {
                dis[u] = di, nf[u] = __uint2float_rn(num);
                num += r32, di += q32;
                if (num >= to) num -= to, di += 1;
            }
#pragma unroll
            for (int u = 0; u < H; u++) x0[u] = __ldg(base_f + dis[u]), x1[u] = __ldg(base_f + dis[u] + 1);
#pragma unroll
            for (int u = 0; u < H; u++) {
                float v = lerp_rcp(gains<NOGAIN>(x0[u], pre, n_pre), gains<NOGAIN>(x1[u], pre, n_pre), nf[u], den_f, rcp_den);
                out[32 * (h + u)] = gains<NOGAIN>(v, mid, n_mid);
            }
        }
        return;
    }
#pragma unroll 1
    for (int h = 0; h < U; h += H) {
        uint32_t dis[H];
        float nf[H], x0[H], x1[H];
#pragma unroll
        for (int u = 0; u < H; u++) {
            dis[u] = di, nf[u] = __uint2float_rn(num);
            num += r32, di += q32;
            if (num >= to) num -= to, di += 1;
        }
#pragma unroll
        for (int u = 0; u < H; u++) {
            x0[u] = 0.0f, x1[u] = 0.0f;
            if (lane + 32u * (uint32_t)(h + u) < n) {
                if (F32) {
                    x0[u] = __ldg(base_f + dis[u]);
                    if (dis[u] < lim) x1[u] = __ldg(base_f + dis[u] + 1);
                } else {
                    x0[u] = load_as_f32(r.in, fmt, rt.i0 + dis[u]);
                    if (dis[u] < lim) x1[u] = load_as_f32(r.in, fmt, rt.i0 + dis[u] + 1);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < H; u++) {
            if (lane + 32u * (uint32_t)(h + u) < n) {
                float v = gains<NOGAIN>(x0[u], pre, n_pre);
                if (dis[u] < lim) v = lerp_rcp(v, gains<NOGAIN>(x1[u], pre, n_pre), nf[u], den_f, rcp_den);
                out[32 * (h + u)] = gains<NOGAIN>(v, mid, n_mid);
            }
        }
    }
}

// Stage A for one (row, tile): the whole warp walks the row's active samples and writes them to `dst`
// (dst[t] for tile position t).  dst may be shared memory (biquad variant) — `Store` abstracts it.
template <bool F32, class Store>
__device__ __forceinline__ void row_stage_a_any(const FusedRow& r, const RowTile& rt, uint32_t c_mix, uint32_t n_pre,
                                                uint32_t n_mid, uint32_t lane, Store store) {
    if (rt.lo >= rt.hi) return;
    const void* in = r.in;
    const uint32_t fmt = r.fmt, c_in = r.c_in, mode = r.mode;
    float pre[MAX_GAINS], mid[MAX_GAINS];
#pragma unroll
    for (int k = 0; k < MAX_GAINS; k++) pre[k] = r.pre[k], mid[k] = r.mid[k];
    if (mode == ROW_DIRECT) {
        for (uint32_t t = rt.lo + lane; t < rt.hi; t += 32) {
            float v = load_in<F32>(in, fmt, rt.o0 + (t - rt.lo));
            store(t, apply_gains(apply_gains(v, pre, n_pre), mid, n_mid));
        }
    } else if (mode == ROW_GENERIC) {
        for (uint32_t t = rt.lo + lane; t < rt.hi; t += 32)
            store(t, row_sample_generic<F32>(r, c_mix, n_pre, n_mid, rt.o0 + (t - rt.lo)));
    } else {
        // lanes walk output FRAMES k = lane, lane+32, ... counted from frame n0 (the frame of position lo).
        // U frames per lane are handled per batch: all index math first, then all loads (2*U independent
        // LDGs in flight per lane -- this stage must cover HBM latency by itself), then the arithmetic.
        constexpr int U = 8;
        const uint32_t n_frames = (rt.hi - rt.lo + rt.j0 + c_mix - 1) / c_mix;
        const uint32_t from = r.uni.from, to = r.uni.to, q32 = r.q32, r32 = r.r32;
        const float den_f = r.den_f, rcp_den = r.rcp_den;
        const uint64_t L = r.uni.tail.L;
        const bool lerp_mode = (mode == ROW_LERP);
        uint32_t di = 0, num = 0;
        if (lerp_mode) {
            uint32_t prod = rt.r0 + lane * from;      // from, to <= 2^20 in this mode
            di = prod / to;
            num = prod - di * to;
        }
        for (uint32_t kb = 0; kb < n_frames; kb += 32 * U) {
            uint32_t dis[U], nums[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                dis[u] = lerp_mode ? di : (kb + lane + 32u * (uint32_t)u);
                nums[u] = num;
                if (lerp_mode) {
                    num += r32, di += q32;
                    if (num >= to) num -= to, di += 1;
                }
            }
            for (uint32_t j = 0; j < c_mix; j++) {
                const int c = chan_map(j, c_in);
                float x0[U], x1[U];
                bool itp[U];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const uint32_t k = kb + lane + 32u * (uint32_t)u;
                    const uint64_t i = rt.i0 + dis[u];
                    itp[u] = lerp_mode && (i + 1 < L);
                    x0[u] = 0.0f, x1[u] = 0.0f;
                    if (k < n_frames && c >= 0) {
                        const uint64_t idx = i * c_in + (uint32_t)c;
                        x0[u] = load_in<F32>(in, fmt, idx);
                        if (itp[u]) x1[u] = load_in<F32>(in, fmt, idx + c_in);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const uint32_t k = kb + lane + 32u * (uint32_t)u;
                    const int t = (int)(rt.lo + k * c_mix + j) - (int)rt.j0;
                    if (k >= n_frames || t < (int)rt.lo || t >= (int)rt.hi) continue;
                    float v = 0.0f;
                    if (c >= 0) {
                        v = apply_gains(x0[u], pre, n_pre);
                        if (itp[u]) v = lerp_rcp(v, apply_gains(x1[u], pre, n_pre), __uint2float_rn(nums[u]), den_f, rcp_den);
                    }
                    store((uint32_t)t, apply_gains(v, mid, n_mid));
                }
            }
        }
    }
}

template <bool F32>
__device__ __forceinline__ void row_stage_a(const FusedRow& r, const RowTile& rt, uint32_t c_mix, uint32_t n_pre,
                                            uint32_t n_mid, uint32_t lane, float* row) {
    if (rt.lo >= rt.hi) return;
    if (r.mode == ROW_LERP && c_mix == 1 && r.c_in == 1) {
        if (n_pre == 0 && n_mid == 0) stage_a_mono_lerp<F32, true>(r, rt, n_pre, n_mid, lane, row);
        else stage_a_mono_lerp<F32, false>(r, rt, n_pre, n_mid, lane, row);
        return;
    }
    row_stage_a_any<F32>(r, rt, c_mix, n_pre, n_mid, lane, [&](uint32_t t, float v) { row[t] = v; });
}

// Copy this CTA's rows into shared memory once (row constants are then warp-broadcast LDS, not LDG).
__device__ __forceinline__ void load_rows(FusedRow* s_rows, const FusedRow* rows, uint32_t G) {
    const uint32_t words = G * (uint32_t)(sizeof(FusedRow) / 4);
    const uint32_t* src = reinterpret_cast<const uint32_t*>(rows);
    uint32_t* dst = reinterpret_cast<uint32_t*>(s_rows);
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
}

__device__ __forceinline__ void cta_span(const FusedRow* s_rows, uint32_t G, const FusedArgs& a, uint64_t& lo,
                                         uint64_t& hi) {
    lo = ~0ull, hi = 0;
    for (uint32_t g = 0; g < G; g++) {
        if (s_rows[g].out_len == 0) continue;
        lo = min(lo, s_rows[g].mix_start);
        hi = max(hi, s_rows[g].mix_start + s_rows[g].out_len);
    }
    if (a.direct || a.chain) lo = 0, hi = a.mix_len;   // chain: every CTA hands the running sum on for every tile
}

// Stage C for one tile position: post-gains and the ordered sum over the CTA's rows.
// `full`: every row of the CTA is active over the whole tile (the common interior case) -> no range checks.
template <int NPOST, class TileState>   // NPOST: 0, 1 or -1 (runtime count); TileState begins with {uint32 lo, hi}
__device__ __forceinline__ float mix_rows_n(const float* tile, const TileState* rts, const FusedRow* s_rows, uint32_t G,
                                            uint32_t n_post, uint32_t t, bool full, float acc = 0.0f) {
    if (full) {
#pragma unroll 4
        for (uint32_t g = 0; g < G; g++) {
            float v = tile[g * ROW_STRIDE + t];
            if (NPOST == 1) v = mul(v, s_rows[g].post[0]);
            else if (NPOST < 0) v = apply_gains(v, s_rows[g].post, n_post);
            acc = add(acc, v);
        }
    } else {
        for (uint32_t g = 0; g < G; g++) {
            const uint2 r = *reinterpret_cast<const uint2*>(&rts[g].lo);   // (lo, hi)
            if (t >= r.x && t < r.y) {
                float v = tile[g * ROW_STRIDE + t];
                if (NPOST == 1) v = mul(v, s_rows[g].post[0]);
                else if (NPOST < 0) v = apply_gains(v, s_rows[g].post, n_post);
                acc = add(acc, v);
            }
        }
    }
    return acc;
}
template <class TileState>
__device__ __forceinline__ float mix_rows(const float* tile, const TileState* rts, const FusedRow* s_rows, uint32_t G,
                                          uint32_t n_post, uint32_t t, bool full, float acc0 = 0.0f) {
    if (n_post == 0) return mix_rows_n<0>(tile, rts, s_rows, G, n_post, t, full, acc0);
    if (n_post == 1) return mix_rows_n<1>(tile, rts, s_rows, G, n_post, t, full, acc0);
    return mix_rows_n<-1>(tile, rts, s_rows, G, n_post, t, full, acc0);
}

// Mixer-timeline interval on which every row of the CTA is active: tiles inside it need no range checks.
__device__ __forceinline__ void cta_full_span(const FusedRow* s_rows, uint32_t G, uint64_t& f_lo, uint64_t& f_hi) {
    f_lo = 0, f_hi = ~0ull;
    for (uint32_t g = 0; g < G; g++) {
        f_lo = max(f_lo, s_rows[g].mix_start);
        f_hi = min(f_hi, s_rows[g].mix_start + s_rows[g].out_len);
    }
}

// ---------------------------------------------------------------------------------------------------
// no-biquad variant: stage A (warp per row) -> shared tile -> stage C (thread per position)
// ---------------------------------------------------------------------------------------------------
template <bool F32>
__global__ void __launch_bounds__(256) k_fused_nobiquad(FusedArgs a) {
    extern __shared__ __align__(16) float smem[];
    __shared__ __align__(16) FusedRow s_rows[MAX_G];
    __shared__ RowTile s_rt[MAX_G];
    const uint32_t row0 = blockIdx.x * a.rows_per_cta;
    const uint32_t G = min(a.rows_per_cta, a.n_rows - row0);
    load_rows(s_rows, a.rows + row0, G);
    __syncthreads();
    float* partial = a.partial + (uint64_t)blockIdx.x * a.mix_len;
    uint64_t lo, hi;
    cta_span(s_rows, G, a, lo, hi);
    if (lo >= hi) return;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    float* tile = smem;
    const uint64_t m_begin = lo / TT * TT;
    uint64_t f_lo, f_hi;
    cta_full_span(s_rows, G, f_lo, f_hi);
    for (uint64_t m0 = m_begin + (uint64_t)blockIdx.y * TT; m0 < hi; m0 += (uint64_t)gridDim.y * TT) {
        for (uint32_t g = warp; g < G; g += n_warps) {
            if (lane == 0) row_tile_setup(s_rows[g], a.c_mix, m0, s_rt[g]);
            __syncwarp();
            float* row = tile + g * ROW_STRIDE;
            row_stage_a<F32>(s_rows[g], s_rt[g], a.c_mix, a.n_pre, a.n_mid, lane, row);
        }
        __syncthreads();
        const bool full = m0 >= f_lo && m0 + TT <= f_hi;
        for (uint32_t t = threadIdx.x; t < TT; t += blockDim.x)
            if (m0 + t < a.mix_len) partial[m0 + t] = mix_rows(tile, s_rt, s_rows, G, a.n_post, t, full);
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------
// biquad variant: three-stage software pipeline over shared-memory tiles
// ---------------------------------------------------------------------------------------------------
// C_MIX_STATIC 1: mono mixer (vectorised recurrence), 0: any channel count.
template <bool F32, int C_MIX_STATIC>
__global__ void __launch_bounds__(512, 1) k_fused_biquad(FusedArgs a, uint32_t n_rec_warps) {
    extern __shared__ __align__(16) float smem[];
    __shared__ __align__(16) FusedRow s_rows[MAX_G];
    __shared__ RowTile s_rt[NBUF][MAX_G];
    const uint32_t row0 = blockIdx.x * a.rows_per_cta;
    const uint32_t G = min(a.rows_per_cta, a.n_rows - row0);
    load_rows(s_rows, a.rows + row0, G);
    __syncthreads();
    float* partial = a.partial + (uint64_t)blockIdx.x * a.mix_len;
    const uint32_t c_mix = C_MIX_STATIC ? (uint32_t)C_MIX_STATIC : a.c_mix;
    uint64_t lo, hi;
    cta_span(s_rows, G, a, lo, hi);
    if (lo >= hi) return;
    const uint64_t m_begin = lo / TT * TT;
    const uint32_t n_tiles = (uint32_t)((hi - m_begin + TT - 1) / TT);
    uint64_t f_lo, f_hi;
    cta_full_span(s_rows, G, f_lo, f_hi);

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n_warps = blockDim.x >> 5;
    // The recurrence warps take the HIGHEST warp ids: the sub-partition arbiter prefers high warp ids, and the
    // dependent FMUL->FADD->FADD chain must never wait for an issue slot behind the throughput warps.
    const uint32_t n_par_warps = n_warps - n_rec_warps;
    const bool is_rec = warp >= n_par_warps;
    const uint32_t n_par_threads = n_par_warps * 32;
    const uint32_t par_tid = threadIdx.x;
    const uint32_t par_warp = warp;

    // recurrence lane -> chain (row, channel); state in registers for the whole stream
    const uint32_t chain = (warp - n_par_warps) * 32 + lane;
    const uint32_t ch_row = chain / c_mix, ch_c = chain - ch_row * c_mix;
    const bool chain_on = is_rec && ch_row < G;
    float x1 = 0.f, x2 = 0.f, y1 = 0.f, y2 = 0.f;
    float b0 = 0.f, b1 = 0.f, b2 = 0.f, a1 = 0.f, a2 = 0.f;
    if (chain_on) {
        const FusedRow& r = s_rows[ch_row];
        b0 = r.b0, b1 = r.b1, b2 = r.b2, a1 = r.a1, a2 = r.a2;
    }

    for (uint32_t it = 0; it < n_tiles + 2; it++) {
        if (!is_rec) {
            // ---- stage A on tile `it`: one warp per row ----
            if (it < n_tiles) {
                const uint32_t buf = it % NBUF;
                const uint64_t m0 = m_begin + (uint64_t)it * TT;
                float* tile = smem + (size_t)buf * MAX_G * ROW_STRIDE;
                for (uint32_t g = par_warp; g < G; g += n_par_warps) {
                    if (lane == 0) row_tile_setup(s_rows[g], c_mix, m0, s_rt[buf][g]);
                    __syncwarp();
                    float* row = tile + g * ROW_STRIDE;
                    row_stage_a<F32>(s_rows[g], s_rt[buf][g], c_mix, a.n_pre, a.n_mid, lane, row);
                }
            }
            // ---- stage C on tile `it - 2` ----
            if (it >= 2) {
                const uint32_t kt = it - 2;
                const uint32_t buf = kt % NBUF;
                const uint64_t m0 = m_begin + (uint64_t)kt * TT;
                const float* tile = smem + (size_t)buf * MAX_G * ROW_STRIDE;
                const bool full = m0 >= f_lo && m0 + TT <= f_hi;
                for (uint32_t t = par_tid; t < TT; t += n_par_threads)
                    if (m0 + t < a.mix_len) partial[m0 + t] = mix_rows(tile, s_rt[buf], s_rows, G, a.n_post, t, full);
            }
        } else if (it >= 1 && it <= n_tiles) {
            // ---- stage B on tile `it - 1` ----
            const uint32_t kt = it - 1;
            const uint32_t buf = kt % NBUF;
            if (chain_on) {
                float* row = smem + (size_t)buf * MAX_G * ROW_STRIDE + ch_row * ROW_STRIDE;
                const uint2 act = *reinterpret_cast<const uint2*>(&s_rt[buf][ch_row].lo);
                const uint32_t lo_t = act.x, hi_t = act.y;
                if (C_MIX_STATIC == 1) {
                    uint32_t t = lo_t;
                    for (; t < hi_t && (t & 3); t++) {               // head up to 16-byte alignment
                        float xv = row[t];
                        float y = biquad_fb(a1, a2, biquad_ff(b0, b1, b2, xv, x1, x2), y1, y2);
                        x2 = x1, x1 = xv, y2 = y1, y1 = y;
                        row[t] = y;
                    }
                    float4 nx = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (t + 4 <= hi_t) nx = *reinterpret_cast<const float4*>(row + t);
                    for (; t + 4 <= hi_t; t += 4) {
                        const float4 xv = nx;
                        if (t + 8 <= hi_t) nx = *reinterpret_cast<const float4*>(row + t + 4);   // prefetch next
                        float4 yv;
                        float f0 = biquad_ff(b0, b1, b2, xv.x, x1, x2);
                        float f1 = biquad_ff(b0, b1, b2, xv.y, xv.x, x1);
                        float f2 = biquad_ff(b0, b1, b2, xv.z, xv.y, xv.x);
                        float f3 = biquad_ff(b0, b1, b2, xv.w, xv.z, xv.y);
                        yv.x = biquad_fb(a1, a2, f0, y1, y2);
                        yv.y = biquad_fb(a1, a2, f1, yv.x, y1);
                        yv.z = biquad_fb(a1, a2, f2, yv.y, yv.x);
                        yv.w = biquad_fb(a1, a2, f3, yv.z, yv.y);
                        x2 = xv.z, x1 = xv.w, y2 = yv.z, y1 = yv.w;
                        *reinterpret_cast<float4*>(row + t) = yv;
                    }
                    for (; t < hi_t; t++) {
                        float xv = row[t];
                        float y = biquad_fb(a1, a2, biquad_ff(b0, b1, b2, xv, x1, x2), y1, y2);
                        x2 = x1, x1 = xv, y2 = y1, y1 = y;
                        row[t] = y;
                    }
                } else {
                    // chain (row, c): positions whose mixer channel is c.  Streams join on a frame boundary
                    // (mixer.rs:175-183) so channel == (m0 + t) % c_mix == (local index) % c_mix.
                    const uint64_t m0 = m_begin + (uint64_t)kt * TT;
                    uint32_t ph = (uint32_t)((m0 + lo_t) % c_mix);
                    uint32_t t = lo_t + (ch_c + c_mix - ph) % c_mix;
                    for (; t < hi_t; t += c_mix) {
                        float xv = row[t];
                        float y = biquad_fb(a1, a2, biquad_ff(b0, b1, b2, xv, x1, x2), y1, y2);
                        x2 = x1, x1 = xv, y2 = y1, y1 = y;
                        row[t] = y;
                    }
                }
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------
// HOT variant (BASELINE cfg3 and its relatives): every row is an f32 source with the mixer's channel count
// (mono or stereo), same rate or linear interpolation with from/to <= 1.2, at most one biquad.
// Same three-stage pipeline, plus a fourth, asynchronous stage in front:
//   L  tile k+2 : each row's input window (<= TT*from/to + 3 frames) is fetched by the bulk-copy engine
//                 (cp.async.bulk global -> shared, completion counted on an mbarrier), two tiles ahead,
//                 so stage A never touches global memory and never waits for HBM latency.
// 1024 threads, one loop per role: 21 stage-A warps (one row each, up to eleven take a second row), the loader warp,
// the recurrence warp alone on its SM sub-partition, stage C on two warps of the stage-A sub-partitions.
// ---------------------------------------------------------------------------------------------------
constexpr int NWIN = 3;                 // input-window ring (tile k .. k+2)
constexpr int WSTRIDE = 320;            // floats per row window (>= 3 + TT*from/to + 3, multiple of 4): from/to <= 1.2
constexpr int WSTRIDE_NARROW = 244;     // the same for from/to <= 0.93 (44.1 -> 48 kHz needs 241): 32 mono rows fit in shared memory
constexpr int NHT = 5;                  // per-(row,tile) index-state ring: written 2 tiles ahead, read until stage C

struct HotTile {
    uint32_t lo, hi;       // active tile positions
    uint32_t r0;           // (n0 * from) mod to at position lo
    uint32_t woff;         // i0 & 3: offset of frame i0 inside the 16-byte aligned window
    uint64_t i0;           // left input frame of position lo
    uint32_t lim;          // frames (relative to i0) that still have a right neighbour: interpolate iff di < lim
    uint32_t interior;     // full tile of an interpolated row, every tap inside the stream: blocked fast path
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// CTA-wide barrier reached from the role-specialised loops (every warp executes the same number of them)
__device__ __forceinline__ void cta_bar() { asm volatile("bar.sync 0;" ::: "memory"); }
#ifdef RB_HOT_TIMING
// Instrumented build (tools/hot_timing.py): cycles each warp spends working / waiting at the tile barrier.
__device__ unsigned long long g_hot_timing[32][4];   // work, barrier, window wait, -
// bit 0: no stage A, bit 1: no recurrence, bit 2: no stage C, bit 3: no second rows, bit 4: conflict-free window addresses, bit 5:
// no range check, bit 6: no stage-A t stores (results are wrong).  In constant memory: read-only to the kernel, so the compiler
// may keep it in a uniform register across the shared-memory stores of stage A.
__constant__ int g_hot_skip;
#define HOT_SKIP(bit) (g_hot_skip_v & (bit))
#define HOT_TIMING_DECL long long tw_ = 0, tb_ = 0, tm_ = 0, tt0_ = clock64(), tt1_ = 0; const int g_hot_skip_v = g_hot_skip;
#define HOT_MBAR_WAIT(bar_, ph_) do { const long long m0_ = clock64(); mbar_wait(bar_, ph_); tm_ += clock64() - m0_; } while (0)
// BAR.SYNC.DEFER_BLOCKING lets the warp run on past the barrier until its next shared-memory access, so the wait is
// made visible with a dependent branch on a volatile shared load (always zero) before the clock is read again.
__device__ __forceinline__ void hot_timing_fence() {
    uint32_t d;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(d) : "r"(0u) : "memory");
    if (d == 0xdeadbeefu) __trap();
}
#define HOT_BAR()                      \
    do {                               \
        hot_timing_fence();            \
        tt1_ = clock64();              \
        cta_bar();                     \
        hot_timing_fence();            \
        const long long t2_ = clock64(); \
        tw_ += tt1_ - tt0_, tb_ += t2_ - tt1_, tt0_ = t2_; \
    } while (0)
#define HOT_TIMING_END                                                        \
    if ((threadIdx.x & 31) == 0) {                                            \
        atomicAdd(&g_hot_timing[threadIdx.x >> 5][0], (unsigned long long)tw_); \
        atomicAdd(&g_hot_timing[threadIdx.x >> 5][1], (unsigned long long)tb_); \
        atomicAdd(&g_hot_timing[threadIdx.x >> 5][2], (unsigned long long)tm_); \
    }
#else
#define HOT_SKIP(bit) false
#define HOT_MBAR_WAIT(bar_, ph_) mbar_wait(bar_, ph_)
#define HOT_TIMING_DECL
#define HOT_BAR() cta_bar()
#define HOT_TIMING_END
#endif
// Stage-A outcomes, counted in row-tiles by the instrumented build -DRB_HOT_PATHS (tests/test_hot_rows_gpu.py), so that a test can
// tell which paths of stage A it ran.  A row-tile ends in exactly one of PAIR, SOLO, REDO and STRIDED; PAIR_FAILED counts the
// row-tiles of a failed pair vote, which then run solo and are counted again there.
enum { HOT_PATH_PAIR = 0, HOT_PATH_PAIR_FAILED, HOT_PATH_SOLO, HOT_PATH_REDO, HOT_PATH_STRIDED, HOT_PATH_N = 8 };
#ifdef RB_HOT_PATHS
__device__ unsigned long long g_hot_paths[HOT_PATH_N];
#define HOT_PATH(k_, n_)                                                                     \
    do {                                                                                     \
        if ((threadIdx.x & 31) == 0) atomicAdd(&g_hot_paths[k_], (unsigned long long)(n_)); \
    } while (0)
#else
#define HOT_PATH(k_, n_) do { } while (0)
#endif

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D bulk copy global -> shared through the TMA/bulk-copy engine; completes `bytes` on the mbarrier.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Index state of (row, tile) -- incremental from the previous tile when that one was a full interior tile.
// C = channels (source == mixer): positions are flat interleaved samples, i0 / r0 / qT / q32 count FRAMES.
template <int C>
__device__ __forceinline__ void hot_tile_setup(const FusedRow& r, uint64_t m0, const HotTile* prev, HotTile& ht) {
    const uint64_t s = r.mix_start, e = r.mix_start + r.out_len;
    const uint64_t lo = m0 > s ? m0 : s, hi = (m0 + TT) < e ? (m0 + TT) : e;
    ht.lo = ht.hi = 0, ht.r0 = 0, ht.woff = 0, ht.i0 = 0, ht.lim = 0, ht.interior = 0;
    if (lo >= hi) return;
    ht.lo = (uint32_t)(lo - m0), ht.hi = (uint32_t)(hi - m0);
    if (prev && prev->lo == 0 && prev->hi == (uint32_t)TT && ht.lo == 0) {
        uint32_t rr = prev->r0 + r.rT;
        uint64_t ii = prev->i0 + r.qT;
        if (rr >= r.uni.to) rr -= r.uni.to, ii += 1;
        ht.r0 = rr, ht.i0 = ii;
    } else {
        const uint64_t prod = ((lo - s) / C) * (uint64_t)r.uni.from;   // streams join and tiles start on frame boundaries
        ht.i0 = prod / r.uni.to;
        ht.r0 = (uint32_t)(prod - ht.i0 * r.uni.to);
    }
    ht.woff = (uint32_t)((ht.i0 * C) & 3ull);
    const uint64_t remain = r.uni.tail.L - 1 - ht.i0;
    ht.lim = remain > 0x7fffffffull ? 0x7fffffffu : (uint32_t)remain;
    // the last frame a full tile touches is i0 + floor((r0 + (TT/C - 1) * from) / to) <= i0 + qT + 1
    ht.interior = r.mode == ROW_LERP && ht.hi - ht.lo == (uint32_t)TT && r.qT + 2 < ht.lim;
}

// Stage L for one (row, tile): arm the stage barrier and launch the bulk copy of the input window.
template <int C>
__device__ __forceinline__ void hot_issue_window(const FusedRow& r, const HotTile& ht, float* win, uint64_t* bar) {
    if (ht.lo >= ht.hi) {
        mbar_arrive(bar);
        return;
    }
    const uint32_t n = ht.hi - ht.lo;
    const uint64_t L = r.uni.tail.L;
    (void)n;
    uint64_t taps = (uint64_t)r.qT + 3;          // >= floor((r0 + (TT-1)*from)/to) + 2 because r0 < to
    if (ht.i0 + taps > L) taps = L - ht.i0;
    const uint32_t floats = ht.woff + (uint32_t)taps * C;
    const uint32_t bytes = (floats * 4u + 15u) & ~15u;                  // <= 12 bytes into the row's 16-byte tail pad
    const float* src = (const float*)r.in + (ht.i0 * C - ht.woff);
    mbar_arrive_expect_tx(bar, bytes);
    bulk_g2s(win, src, bytes, bar);
}

// Stage A for one (row, tile) out of the shared-memory window.
// Full interior tiles use a BLOCKED layout: lane l owns the P = TT/32 consecutive positions P*l .. P*l+P-1
// (P/C frames), so that
//   * the index state advances by ONE frame per step -- kept as a float numerator (exact, < 2^24) and a word
//     offset into the window: FADD, FSETP, two predicated adds per frame;
//   * the feed-forward half of the biquad, t[n] = (b0*x[n] + b1*x[n-1]) + b2*x[n-2] (same three roundings as the
//     reference; it does not depend on y), finds its left neighbours in the lane's own registers -- only the
//     first 2C positions take them from lane l-1 by shuffle, and lane 0 from `xtail`, the previous tile's last 2C
//     x values (replicated in every lane);
//   * t leaves with two 16-byte stores.  x itself never touches shared memory.
// (lane_q, lane_r) = divmod(lane * (P/C) * from, to), computed once per kernel by the row's warp; r.q32 / r.r32 =
// divmod(from, to), the per-frame step.
// The exact-division fast path is used optimistically: a per-lane flag collects "operand outside the guarded
// range" and ONE warp vote per row-tile decides whether the tile is redone with IEEE divisions.
// A single warp issues roughly one instruction every two cycles, so the recurrence warp can only stay on its
// 12-cycle dependent chain if it executes nothing but  y = (t - a1*y1) - a2*y2  -- hence t, not x, in the row.
// Partial tiles (stream start / end, same-rate rows, the IEEE redo) take the strided path below: lane l works on
// positions l + 32u, x goes through the row in shared memory, `row[-2C..-1]` are pad slots for the tail.
// HASB = false (no filter in the chain: resample -> gains -> mix): the row receives x itself, there is no tail.
// One interior sample: lerp of the taps (x0, x1) at numerator nfc with the exact-reciprocal division; `bad` collects
// "operand outside the guarded range".
template <bool NOGAIN>
__device__ __forceinline__ float hot_lerp(float x0, float x1, float nfc, float den_f, float rcp_den, const float* pre, uint32_t n_pre,
                                          const float* mid, uint32_t n_mid, bool& bad) {
    const float a0 = gains<NOGAIN>(x0, pre, n_pre), a1 = gains<NOGAIN>(x1, pre, n_pre);
    const float m = mul(sub(a1, a0), nfc);
    const float q0 = mul(m, rcp_den);
    const float q = __fmaf_rn(__fmaf_rn(-q0, den_f, m), rcp_den, q0);
    // guarded range as one unsigned compare on the exponent field: 2^-100 <= |m| < 2^100; m == 0
    // (also outside) yields q = m = +-0 exactly as the division would
    const uint32_t e = __float_as_uint(m) & 0x7fffffffu;
    const bool in_range = e - 0x0d800000u < 0x64000000u;
#ifdef RB_HOT_TIMING
    if (!(g_hot_skip & 32))               // ablation: no range check
#endif
    bad |= !in_range && e != 0u;
    return gains<NOGAIN>(add(a0, in_range ? q : m), mid, n_mid);
}
// Interior tile, after the vote: the lane's P consecutive x values -> t (the feed-forward half; x itself without a filter)
// -> two 16-byte stores at row[P*lane ..].  xtail takes the tile's last 2C x values.
template <int C, bool HASB>
__device__ __forceinline__ void hot_ff_store(float b0, float b1, float b2, const float (&xv)[TT / 32], float (&xtail)[2 * C],
                                             uint32_t lane, float* __restrict__ row) {
    constexpr int P = TT / 32;
    float tv[P];
    if constexpr (HASB) {
        float pv[2 * C];
#pragma unroll
        for (int j = 0; j < 2 * C; j++) {
            const float up = __shfl_up_sync(0xffffffffu, xv[P - 2 * C + j], 1);
            pv[j] = lane == 0 ? xtail[j] : up;
        }
#pragma unroll
        for (int j = 0; j < 2 * C; j++) xtail[j] = __shfl_sync(0xffffffffu, xv[P - 2 * C + j], 31);
#pragma unroll
        for (int u = 0; u < P; u++) {
            const float xm1 = u >= C ? xv[u >= C ? u - C : 0] : pv[C + u < 2 * C ? C + u : 0];
            const float xm2 = u >= 2 * C ? xv[u >= 2 * C ? u - 2 * C : 0] : pv[u < 2 * C ? u : 0];
            tv[u] = biquad_ff(b0, b1, b2, xv[u], xm1, xm2);
        }
    } else {
#pragma unroll
        for (int u = 0; u < P; u++) tv[u] = xv[u];
    }
#ifdef RB_HOT_TIMING
    if (g_hot_skip & 64) {   // ablation: no t stores (a test that almost never passes keeps the feed-forward live)
        uint32_t h = 0;
#pragma unroll
        for (int u = 0; u < P; u++) h ^= __float_as_uint(tv[u]);
        if (h != 0x7fbadbadu) return;
    }
#endif
    // Lanes l and l + 4 cover the same banks with 16-byte stores at a 32-byte lane stride.  In the mono kernel the lanes with
    // (l >> 2) & 1 write their second 16 bytes first, so that each 8-lane phase of an STS.128 covers all 32 banks once.
    static_assert(P == 8, "two 16-byte stores per lane");
    const float4 v0 = make_float4(tv[0], tv[1], tv[2], tv[3]), v1 = make_float4(tv[4], tv[5], tv[6], tv[7]);
    const bool sw = C == 1 && ((lane >> 2) & 1u);
    float4* o = reinterpret_cast<float4*>(row + P * lane);
    o[sw ? 1 : 0] = sw ? v1 : v0;
    o[sw ? 0 : 1] = sw ? v0 : v1;
}

template <bool NOGAIN, int C, bool HASB>
__device__ __forceinline__ void hot_stage_a(const FusedRow& r, const HotTile& ht, uint32_t n_pre, uint32_t n_mid,
                                            uint32_t lane, uint32_t lane_q, uint32_t lane_r, float (&xtail)[2 * C],
                                            const float* __restrict__ win, float* __restrict__ row) {
    constexpr int U = TT / 32, P = TT / 32, F = P / C;
    const uint32_t n = ht.hi - ht.lo;
    const uint32_t to = r.uni.to;
    const float den_f = r.den_f, rcp_den = r.rcp_den;
    const float b0 = r.b0, b1 = r.b1, b2 = r.b2;
    const uint32_t lim = ht.lim;
    const float* pre = r.pre;
    const float* mid = r.mid;
    const bool pass = r.mode != ROW_LERP;   // same-rate rows: x[n] = in[n], no interpolation (from = to = 1 in the row)
    bool done = false;
    {
        uint32_t num = ht.r0 + lane_r;
        uint32_t di = lane_q;
        if (num >= to) num -= to, di += 1;
        const bool interior = ht.interior != 0;   // warp-uniform (planned by the loader): the vote below needs the whole warp
        if (interior) {
            const float* __restrict__ w = win + ht.woff + di * C;
#ifdef RB_HOT_TIMING
            if (g_hot_skip & 16) w = win + lane;          // ablation: conflict-free (wrong) window addresses
#endif
            const uint32_t step_w = r.q32 * C;            // whole frames per output frame, in words
            const float r1f = __uint2float_rn(r.r32);
            float nf = __uint2float_rn(num);
            bool bad = false;
            float xv[P];
            if (step_w == 0) {
                // from < to: only the right tap is loaded, the left one is the previous frame's right (index moved) or left tap
                // (hot_stage_a_pair)
                float x0[C], x1[C];
#pragma unroll
                for (int c = 0; c < C; c++) x0[c] = w[c], x1[c] = w[C + c];
#pragma unroll
                for (int f = 0; f < F; f++) {
                    const float nfc = nf;
                    nf = add(nf, r1f);
                    const bool carry = nf >= den_f;
                    if (carry) nf = sub(nf, den_f), w += C;
#pragma unroll
                    for (int c = 0; c < C; c++) xv[f * C + c] = hot_lerp<NOGAIN>(x0[c], x1[c], nfc, den_f, rcp_den, pre, n_pre, mid, n_mid, bad);
                    if (f + 1 < F) {
#pragma unroll
                        for (int c = 0; c < C; c++) {
                            const float x2 = w[C + c];
                            x0[c] = carry ? x1[c] : x0[c];
                            x1[c] = x2;
                        }
                    }
                }
            } else {
#pragma unroll
                for (int f = 0; f < F; f++) {
                    float x0[C], x1[C];
#pragma unroll
                    for (int c = 0; c < C; c++) x0[c] = w[c], x1[c] = w[C + c];
                    const float nfc = nf;
                    nf = add(nf, r1f);
                    w += step_w;
                    if (nf >= den_f) nf = sub(nf, den_f), w += C;
#pragma unroll
                    for (int c = 0; c < C; c++) xv[f * C + c] = hot_lerp<NOGAIN>(x0[c], x1[c], nfc, den_f, rcp_den, pre, n_pre, mid, n_mid, bad);
                }
            }
            if (!__any_sync(0xffffffffu, bad)) {
                hot_ff_store<C, HASB>(b0, b1, b2, xv, xtail, lane, row);
                done = true;
            }
            // else: some operand was denormal / huge / NaN: redo this row-tile with IEEE divisions
            HOT_PATH(done ? HOT_PATH_SOLO : HOT_PATH_REDO, 1);
        } else {
            HOT_PATH(HOT_PATH_STRIDED, 1);
        }
    }
    if (done) return;
    // strided path: partial tiles, end of stream, same-rate rows, or the rare IEEE-division redo
    const uint32_t fs = (32u / C) * r.uni.from;            // frames step of 32 positions
    const uint32_t q32 = fs / to, r32 = fs - q32 * to;
    const uint32_t pl = (lane / C) * r.uni.from;
    uint32_t di = pl / to;
    uint32_t num = ht.r0 + (pl - di * to);
    if (num >= to) num -= to, di += 1;
    const float* __restrict__ w = win + ht.woff + (lane % C);   // this lane's channel
    float* __restrict__ out = row + ht.lo + lane;
    // x of the 2C positions before the first active one: zeros when the stream starts in this tile, else the tail
    const bool first = ht.i0 == 0 && ht.r0 == 0;
    if constexpr (HASB) {
#pragma unroll
        for (int j = 0; j < 2 * C; j++)
            if (lane == (uint32_t)j) row[(int)ht.lo - 2 * C + j] = first ? 0.0f : xtail[j];
    }
#pragma unroll 1
    for (int u = 0; u < U; u++) {
        if (lane + 32u * (uint32_t)u < n) {
            float v = gains<NOGAIN>(w[di * C], pre, n_pre);
            if (!pass && di < lim) v = lerp_f(v, gains<NOGAIN>(w[(di + 1) * C], pre, n_pre), __uint2float_rn(num), den_f);
            out[32 * u] = gains<NOGAIN>(v, mid, n_mid);
        }
        num += r32, di += q32;
        if (num >= to) num -= to, di += 1;
    }
    if constexpr (!HASB) return;
    __syncwarp();
    float xv[U], xm1[U], xm2[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
        xv[u] = xm1[u] = xm2[u] = 0.0f;
        if (lane + 32u * (uint32_t)u < n) xv[u] = out[32 * u], xm1[u] = out[32 * u - C], xm2[u] = out[32 * u - 2 * C];
    }
    // new tail = x at the last 2C active positions (a one-frame tile shifts the old tail in from the pad slots)
#pragma unroll
    for (int j = 0; j < 2 * C; j++) xtail[j] = row[(int)ht.hi - 2 * C + j];
    __syncwarp();
#pragma unroll
    for (int u = 0; u < U; u++)
        if (lane + 32u * (uint32_t)u < n) out[32 * u] = biquad_ff(b0, b1, b2, xv[u], xm1[u], xm2[u]);
}

// Stage A for the two mono rows of one warp when their tiles are in phase: both interior, the same rate pair (hence the same
// lane constants) and the same r0.  Numerator and window offset then advance identically for both rows, so ONE index walk
// (FADD, FSETP, the predicated adds, the address) serves both windows, and one vote covers both.  The two rows' loads and
// arithmetic interleave; each row keeps its own window, gains, taps and tail.  Returns false when the vote fails: the caller
// then runs each row on its own, which redoes the tile with IEEE divisions.
template <bool NOGAIN, bool HASB>
__device__ __forceinline__ bool hot_stage_a_pair(const FusedRow& ra, const FusedRow& rb, const HotTile& ha, const HotTile& hb,
                                                 uint32_t n_pre, uint32_t n_mid, uint32_t lane, uint32_t lane_q, uint32_t lane_r,
                                                 float (&tail_a)[2], float (&tail_b)[2], const float* win_a, const float* win_b,
                                                 float* row_a, float* row_b) {
    constexpr int P = TT / 32;
    const uint32_t to = ra.uni.to;
    const float den_f = ra.den_f, rcp_den = ra.rcp_den;
    uint32_t num = ha.r0 + lane_r;
    uint32_t di = lane_q;
    if (num >= to) num -= to, di += 1;
    const float* w = win_a + ha.woff + di;
    const int db = (int)((win_b + hb.woff) - (win_a + ha.woff));   // row b's taps relative to row a's (warp-uniform)
#ifdef RB_HOT_TIMING
    if (g_hot_skip & 16) w = win_a + lane;        // ablation: conflict-free (wrong) window addresses
#endif
    const uint32_t step_w = ra.q32;
    const float r1f = __uint2float_rn(ra.r32);
    float nf = __uint2float_rn(num);
    bool bad = false;
    float xa[P], xb[P];
    if (step_w == 0) {
        // from < to (q32 == 0): the window index moves by 0 or 1 word per frame.  When it moves, the next frame's left tap is this
        // frame's right tap; when it stays, both taps stay.  So only the right tap is loaded: one LDS per frame and row.
        float a0 = w[0], a1 = w[1], b0 = w[db], b1 = w[db + 1];
#pragma unroll
        for (int f = 0; f < P; f++) {
            const float nfc = nf;
            nf = add(nf, r1f);
            const bool carry = nf >= den_f;
            if (carry) nf = sub(nf, den_f), w += 1;
            xa[f] = hot_lerp<NOGAIN>(a0, a1, nfc, den_f, rcp_den, ra.pre, n_pre, ra.mid, n_mid, bad);
            xb[f] = hot_lerp<NOGAIN>(b0, b1, nfc, den_f, rcp_den, rb.pre, n_pre, rb.mid, n_mid, bad);
            if (f + 1 < P) {
                const float a2 = w[1], b2 = w[db + 1];
                a0 = carry ? a1 : a0, b0 = carry ? b1 : b0;
                a1 = a2, b1 = b2;
            }
        }
    } else {
#pragma unroll
        for (int f = 0; f < P; f++) {
            const float a0 = w[0], a1 = w[1], b0 = w[db], b1 = w[db + 1];
            const float nfc = nf;
            nf = add(nf, r1f);
            w += step_w;
            if (nf >= den_f) nf = sub(nf, den_f), w += 1;
            xa[f] = hot_lerp<NOGAIN>(a0, a1, nfc, den_f, rcp_den, ra.pre, n_pre, ra.mid, n_mid, bad);
            xb[f] = hot_lerp<NOGAIN>(b0, b1, nfc, den_f, rcp_den, rb.pre, n_pre, rb.mid, n_mid, bad);
        }
    }
    if (__any_sync(0xffffffffu, bad)) return false;
    hot_ff_store<1, HASB>(ra.b0, ra.b1, ra.b2, xa, tail_a, lane, row_a);
    hot_ff_store<1, HASB>(rb.b0, rb.b1, rb.b2, xb, tail_b, lane, row_b);
    return true;
}

// Warp roles (32 warps; sub-partition = warp % 4).  Measured: the recurrence warp must have its sub-partition
// to itself.  Its dependent chain (FMUL -> FFMA -> FFMA, 12.9 cycles per sample when alone) needs every issue slot
// on time: with the loader as its neighbour it ran at 16.4 cycles per sample, with stage-A warps at twice that.
//   warp 31                  recurrence (stage B), alone on sub-partition 3 (warps 3,7,..,27 idle)
//   warp 30                  loader (stage L, lane = row)
//   the other 23 warps with warp % 4 != 3: stage A, slot = (warp/4)*3 + warp%4 (sub-partition = slot % 3).
//   Default launch: stage C runs on slots {6, 7} (sub-partitions 0 and 1), which own no row.  The other 21 slots own
//   rows 0..20 in slot order, and rows 21..31 are the second rows of slots {0,3,9,12 | 1,4,10,13 | 2,5,8}, taken in the
//   order 0,1,2,3,4,5,9,10,8,12,13: sub-partitions 0 and 1 carry 11 rows and half of stage C each, sub-partition 2
//   carries 10 rows and the loader.  A warp with two mono rows walks both in one pass when their tiles are in phase
//   (hot_stage_a_pair), so a second row costs less than a first.
//   Chain mode: stage C runs on warps 3 and 7 (below), all 23 slots own rows 0..22, and rows 23..31 are the second rows of
//   slots {0,3,9 | 1,4,10 | 2,5,8} in the same order: 11, 11 and 10 rows + loader.
// 32 rows need the narrow window stride (WSTRIDE_NARROW) to fit in shared memory; with the wide one a CTA takes 28.  On the
// 132 SMs of an H100, 32 rows put the 4096 streams of the benchmarked batch into ONE wave of 128 CTAs (28 rows: 147 CTAs,
// two waves, each walking the whole recurrence).
constexpr uint32_t HOT_MAX_ROWS = 28;          // 21 slots + 7 second rows (wide windows)
constexpr uint32_t HOT_MAX_ROWS_NARROW = 32;   // 21 slots + 11 second rows (mono, narrow windows)
constexpr uint32_t HOT_MAX_ROWS_STEREO = 28;   // 56 chains: a second recurrence warp (27, same sub-partition) takes rows 16..27
constexpr uint32_t HOT_REC_WARP2 = 27;
constexpr uint32_t HOT_REC_WARP = 31, HOT_LOAD_WARP = 30;
__device__ __forceinline__ int hot_row_slot(uint32_t warp) {
    if ((warp & 3u) == 3u || warp == HOT_LOAD_WARP) return -1;
    return (int)((warp >> 2) * 3u + (warp & 3u));   // 0..22
}
// first row of a slot, or -1 (the stage-C slots of the default launch)
template <bool CHAIN>
__device__ __forceinline__ int hot_first_row(int slot) {
    return CHAIN || slot < 6 ? slot : slot < 8 ? -1 : slot - 2;
}
// second row of a slot (rows beyond the slots' first rows), or -1
template <bool CHAIN>
__device__ __forceinline__ int hot_second_row(int slot) {
    constexpr int base = CHAIN ? 23 : 21;
    const int j = slot < 6 ? slot : slot == 9 ? 6 : slot == 10 ? 7 : slot == 8 ? 8 : slot == 12 ? 9 : slot == 13 ? 10 : -1;
    return j < 0 || base + j >= (int)HOT_MAX_ROWS_NARROW ? -1 : base + j;
}
// Stage C of the HOT kernel: one thread sums FOUR consecutive tile positions over the CTA's rows (row order =
// the mixer's insertion order), 16-byte loads of y, the post-gain applied on the fly.  64 threads cover a tile.
template <int NPOST>
__device__ __forceinline__ float4 hot_mix4_full(const float* tile, const FusedRow* s_rows, uint32_t G, uint32_t n_post, uint32_t t4,
                                                float4 acc) {
#pragma unroll 4
    for (uint32_t g = 0; g < G; g++) {
        float4 v = *reinterpret_cast<const float4*>(tile + g * ROW_STRIDE + t4);
        if (NPOST == 1) {
            const float pg = s_rows[g].post[0];
            v.x = mul(v.x, pg), v.y = mul(v.y, pg), v.z = mul(v.z, pg), v.w = mul(v.w, pg);
        } else if (NPOST < 0) {
            v.x = apply_gains(v.x, s_rows[g].post, n_post), v.y = apply_gains(v.y, s_rows[g].post, n_post);
            v.z = apply_gains(v.z, s_rows[g].post, n_post), v.w = apply_gains(v.w, s_rows[g].post, n_post);
        }
        acc.x = add(acc.x, v.x), acc.y = add(acc.y, v.y), acc.z = add(acc.z, v.z), acc.w = add(acc.w, v.w);
    }
    return acc;
}
// Chain mode (RB_MIX_EXACT_ORDER): the sum of a tile starts from the row CTA c - 1 wrote for it (the running sum over all earlier
// streams) instead of +0.0, so the last CTA's row is the reference's sequential sum over every stream.  A CTA only ever waits for
// the CTA in front of it, which holds an earlier ticket and is therefore already running: no co-residency is needed.
// The hand-over carries its own flag: a row of the chain is an array of (value, tag) pairs written and read as single 8-byte
// accesses (single-copy atomic), tag = render number and tile -- the reader polls the DATA until the tag is the one it expects.
// One L2 round trip per hop, no fences, no separate flag (the first version -- release store of a tile counter behind a fenced row,
// acquire poll, then the carry load -- cost 4.8 us per tile and CTA: two fences and three dependent round trips).
// one 64-bit access each (naturally aligned: single-copy atomic -- a .v2.u32 access is formally two scalar accesses)
__device__ __forceinline__ uint2 ld_relaxed_v2(const uint2* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return make_uint2((uint32_t)v, (uint32_t)(v >> 32));
}
__device__ __forceinline__ void st_relaxed_v2(uint2* p, uint2 v) {
    const unsigned long long w = (unsigned long long)v.x | ((unsigned long long)v.y << 32);
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ void hot_mix4(const float* tile, const HotTile* hts, const FusedRow* s_rows, uint32_t G,
                                         uint32_t n_post, uint32_t t4, bool full, uint64_t m0, uint64_t mix_len,
                                         float* __restrict__ partial, bool chain = false, const uint2* carry_row = nullptr,
                                         uint2* tagged_row = nullptr, uint32_t tag = 0) {
    if (m0 + t4 >= mix_len) return;
    const uint32_t n_here = (uint32_t)min((uint64_t)4, mix_len - (m0 + t4));
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (carry_row) {
        const uint2* c = carry_row + m0 + t4;
        uint2 w[4];
        uint32_t spins = 0;
        while (true) {
            bool ok = true;
#pragma unroll
            for (uint32_t k = 0; k < 4; k++)
                if (k < n_here) w[k] = ld_relaxed_v2(c + k), ok = ok && w[k].y == tag;
            if (ok) break;
            if (++spins > (1u << 22)) __trap();      // the CTA in front never arrived: fail loudly instead of hanging the device
        }
        acc.x = __uint_as_float(w[0].x);
        if (n_here > 1) acc.y = __uint_as_float(w[1].x);
        if (n_here > 2) acc.z = __uint_as_float(w[2].x);
        if (n_here > 3) acc.w = __uint_as_float(w[3].x);
    }
    if (full) {
        acc = n_post == 0 ? hot_mix4_full<0>(tile, s_rows, G, n_post, t4, acc)
              : n_post == 1 ? hot_mix4_full<1>(tile, s_rows, G, n_post, t4, acc)
                            : hot_mix4_full<-1>(tile, s_rows, G, n_post, t4, acc);
    } else {
        acc.x = mix_rows(tile, hts, s_rows, G, n_post, t4, false, acc.x);
        acc.y = mix_rows(tile, hts, s_rows, G, n_post, t4 + 1, false, acc.y);
        acc.z = mix_rows(tile, hts, s_rows, G, n_post, t4 + 2, false, acc.z);
        acc.w = mix_rows(tile, hts, s_rows, G, n_post, t4 + 3, false, acc.w);
    }
    if (chain && tagged_row) {     // hand the running sum on: (value, tag) pairs
        uint2* o = tagged_row + m0 + t4;
        st_relaxed_v2(o, make_uint2(__float_as_uint(acc.x), tag));
        if (n_here > 1) st_relaxed_v2(o + 1, make_uint2(__float_as_uint(acc.y), tag));
        if (n_here > 2) st_relaxed_v2(o + 2, make_uint2(__float_as_uint(acc.z), tag));
        if (n_here > 3) st_relaxed_v2(o + 3, make_uint2(__float_as_uint(acc.w), tag));
        return;
    }
    float* o = partial + m0 + t4;
    if (n_here == 4 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
        *reinterpret_cast<float4*>(o) = acc;
    } else {
        o[0] = acc.x;
        if (n_here > 1) o[1] = acc.y;
        if (n_here > 2) o[2] = acc.z;
        if (n_here > 3) o[3] = acc.w;
    }
}

// C == 2 (stereo source into a stereo mixer): a row carries two recurrence chains; the recurrence lane is
// (row, channel) and a second recurrence warp on the same sub-partition takes the chains of rows 16..27.
template <int C, bool HASB, bool CHAIN>   // CHAIN: RB_MIX_EXACT_ORDER, an instantiation of its own (the default launch keeps its code: measured)
__global__ void __launch_bounds__(1024, 1) k_fused_hot(FusedArgs a) {
    extern __shared__ __align__(16) float smem[];
    __shared__ __align__(16) FusedRow s_rows[MAX_G];
    __shared__ __align__(8) HotTile s_ht[NHT][MAX_G];
    __shared__ __align__(8) uint64_t s_full[NWIN];
    // chain mode: the CTA's place in the chain is the order in which the CTAs START (a ticket), not blockIdx.x -- a CTA then only
    // ever waits for one that is already running, whatever order the hardware hands the blocks out in
    __shared__ uint32_t s_cta;
    if (CHAIN) {
        if (threadIdx.x == 0) s_cta = atomicAdd(a.flags, 1u) - a.epoch * gridDim.x;
        __syncthreads();
    }
    const uint32_t cta = CHAIN ? s_cta : blockIdx.x;
    const uint32_t row0 = cta * a.rows_per_cta;
    const uint32_t G = min(a.rows_per_cta, a.n_rows - row0);
    load_rows(s_rows, a.rows + row0, G);
    if (threadIdx.x == 0) {
        for (int i = 0; i < NWIN; i++) mbar_init(&s_full[i], G);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    float* tiles = smem;                                               // [NBUF][rows_per_cta][ROW_STRIDE]
    float* wins = smem + (size_t)NBUF * a.rows_per_cta * ROW_STRIDE;   // [NWIN][rows_per_cta][wstride]
    const uint32_t wstride = a.win_stride;
    const size_t tile_sz = (size_t)a.rows_per_cta * ROW_STRIDE, win_sz = (size_t)a.rows_per_cta * wstride;
    float* partial = a.partial + (uint64_t)cta * a.mix_len;
    const uint2* carry_row = nullptr;      // chain: rows of (value, tag) pairs, `partial` is then [n_ctas][mix_len] of those
    uint2* tagged_row = nullptr;
    if (CHAIN) {
        uint2* rows2 = reinterpret_cast<uint2*>(a.partial);
        if (cta + 1 == gridDim.x) partial = a.out;                       // the last CTA writes the mixer output itself
        else tagged_row = rows2 + (uint64_t)cta * a.mix_len;
        if (cta > 0) carry_row = rows2 + (uint64_t)(cta - 1) * a.mix_len;
    }
    uint64_t lo, hi;
    cta_span(s_rows, G, a, lo, hi);
    if (lo >= hi) return;
    uint64_t m_begin = lo / TT * TT;
    uint32_t n_tiles = (uint32_t)((hi - m_begin + TT - 1) / TT);
    if (!HASB && gridDim.y > 1) {
        // no recurrence, no state: the timeline of the row group is cut into gridDim.y independent slices
        const uint32_t t0 = (uint32_t)((uint64_t)n_tiles * blockIdx.y / gridDim.y);
        const uint32_t t1 = (uint32_t)((uint64_t)n_tiles * (blockIdx.y + 1) / gridDim.y);
        if (t0 >= t1) return;
        m_begin += (uint64_t)t0 * TT, n_tiles = t1 - t0;
    }
    uint64_t f_lo, f_hi;
    cta_full_span(s_rows, G, f_lo, f_hi);

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool is_rec = warp == HOT_REC_WARP || (C == 2 && warp == HOT_REC_WARP2), is_loader = warp == HOT_LOAD_WARP;
    const int slot = hot_row_slot(warp);
    // stage C: two warps of their own, 4 positions per thread, so that its loop state is never live beside a row's stage A.
    // Default launch: slots 6 and 7 (sub-partitions 0 and 1).  Chain mode: warps 3 and 7 (idle otherwise; the recurrence warp's
    // sub-partition has issue slots to spare) -- the hand-over is latency, not work, and must not sit behind a row's stage A.
    const int mix_block = CHAIN ? (warp == 3 ? 0 : warp == 7 ? 1 : -1) : (slot == 6 ? 0 : slot == 7 ? 1 : -1);
    const bool nogain = a.n_pre == 0 && a.n_mid == 0;
    // prologue: the loader warp (lane = row) fetches the windows of tiles 0 and 1
    if (is_loader && lane < G) {
        for (uint32_t kt = 0; kt < 2 && kt < n_tiles; kt++) {
            HotTile& ht = s_ht[kt % NHT][lane];
            hot_tile_setup<C>(s_rows[lane], m_begin + (uint64_t)kt * TT, kt ? &s_ht[(kt - 1) % NHT][lane] : nullptr, ht);
            hot_issue_window<C>(s_rows[lane], ht, wins + (kt % NWIN) * win_sz + lane * wstride, &s_full[kt % NWIN]);
        }
    }
    __syncthreads();

    // One loop per role, n_tiles + 2 iterations each, joined by the CTA barrier at the end of every iteration.
    // Ring positions (tile % NBUF, % NWIN, % NHT) are carried incrementally: the role bodies are short enough
    // that a handful of modulo / dispatch instructions per warp and iteration showed up as a third of all issue slots.
    const uint32_t n_iter = n_tiles + 2;
    HOT_TIMING_DECL
    if (is_loader) {
        // ---- stage L on tile it+2: lane g plans and fetches row g's window ----
        uint32_t kw = 2 % NWIN, kh = 2 % NHT, khp = 1;
        for (uint32_t it = 0; it < n_iter; it++) {
            const uint32_t kt = it + 2;
            if (lane < G && kt < n_tiles) {
                HotTile& ht = s_ht[kh][lane];
                hot_tile_setup<C>(s_rows[lane], m_begin + (uint64_t)kt * TT, &s_ht[khp][lane], ht);
                hot_issue_window<C>(s_rows[lane], ht, wins + kw * win_sz + lane * wstride, &s_full[kw]);
            }
            khp = kh;
            kh = kh + 1 == NHT ? 0 : kh + 1;
            kw = kw + 1 == NWIN ? 0 : kw + 1;
            HOT_BAR();
        }
    } else if (is_rec) {
        // ---- stage B on tile it-1 (lane = chain): nothing but y = (t - a1*y1) - a2*y2 ----
        // two latency-bound warps interleave on one sub-partition without slowing each other much
        const uint32_t chain = (warp == HOT_REC_WARP ? 0u : 32u) + lane;
        const uint32_t rec_row = chain / C, rec_ch = chain % C;
        const bool chain_on = rec_row < G;
        float y1 = 0.f, y2 = 0.f, a1 = 0.f, a2 = 0.f;
        if (chain_on) a1 = s_rows[rec_row].a1, a2 = s_rows[rec_row].a2;
        // -1.0 as a run-time value (ptxas would turn fma(p, -1.0, t) back into an FADD)
        const float neg1 = -s_rows[0].den_f / s_rows[0].den_f;
#define FB(t_, y1_, y2_) biquad_fb_chain(a1, a2, t_, y1_, y2_, neg1)
        float* rbase = tiles + rec_row * ROW_STRIDE + HOT_PAD;
        uint32_t kb = 0, kh = 0;
        HOT_BAR();   // it == 0: nothing to do yet
        for (uint32_t it = 1; it < n_iter; it++) {
            if (HASB && it <= n_tiles && chain_on && !HOT_SKIP(2)) {
                float* row = rbase + kb * tile_sz;
                const uint2 act = *reinterpret_cast<const uint2*>(&s_ht[kh][rec_row].lo);
                uint32_t t = act.x;
                const uint32_t hi_t = act.y;
                if constexpr (C == 1) {
                    for (; t < hi_t && (t & 3); t++) {
                        const float y = FB(row[t], y1, y2);
                        y2 = y1, y1 = y;
                        row[t] = y;
                    }
                    float4* p4 = reinterpret_cast<float4*>(row + t);
                    uint32_t n4 = hi_t > t ? (hi_t - t) >> 2 : 0;
                    t += n4 << 2;
                    // 16 samples per step, the next step's four loads issued a whole step (~200 cycles) ahead of their
                    // use: the serial chain never waits on shared memory.  The look-ahead reads at most 64 bytes past
                    // the active span -- the next row, or the window ring that follows the last row.
#define FB4(v_, o_)                          \
    o_.x = FB(v_.x, y1, y2);                 \
    o_.y = FB(v_.y, o_.x, y1);               \
    o_.z = FB(v_.z, o_.y, o_.x);             \
    o_.w = FB(v_.w, o_.z, o_.y);             \
    y2 = o_.z, y1 = o_.w;
                    if (n4 >= 4) {
                        float4 c0 = p4[0], c1 = p4[1], c2 = p4[2], c3 = p4[3];
                        while (n4 >= 8) {
                            const float4 d0 = p4[4], d1 = p4[5], d2 = p4[6], d3 = p4[7];
                            float4 o;
                            FB4(c0, o) p4[0] = o;
                            FB4(c1, o) p4[1] = o;
                            FB4(c2, o) p4[2] = o;
                            FB4(c3, o) p4[3] = o;
                            c0 = p4[8], c1 = p4[9], c2 = p4[10], c3 = p4[11];
                            FB4(d0, o) p4[4] = o;
                            FB4(d1, o) p4[5] = o;
                            FB4(d2, o) p4[6] = o;
                            FB4(d3, o) p4[7] = o;
                            p4 += 8, n4 -= 8;
                        }
                        if (n4 >= 4) {
                            float4 o;
                            FB4(c0, o) p4[0] = o;
                            FB4(c1, o) p4[1] = o;
                            FB4(c2, o) p4[2] = o;
                            FB4(c3, o) p4[3] = o;
                            p4 += 4, n4 -= 4;
                        }
                    }
                    for (; n4; n4--, p4++) {
                        const float4 v = p4[0];
                        float4 o;
                        FB4(v, o) p4[0] = o;
                    }
#undef FB4
                    for (; t < hi_t; t++) {
                        const float y = FB(row[t], y1, y2);
                        y2 = y1, y1 = y;
                        row[t] = y;
                    }
                } else {
                    // interleaved frames: lo / hi are even, this lane owns positions t + rec_ch
                    float* rc = row + rec_ch;
                    if (t < hi_t && (t & 3)) {
                        const float y = FB(rc[t], y1, y2);
                        y2 = y1, y1 = y;
                        rc[t] = y;
                        t += 2;
                    }
                    float4 nx = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (t + 4 <= hi_t) nx = *reinterpret_cast<const float4*>(row + t);
#pragma unroll 2
                    for (; t + 4 <= hi_t; t += 4) {
                        const float4 f = nx;
                        if (t + 8 <= hi_t) nx = *reinterpret_cast<const float4*>(row + t + 4);
                        const float ya = FB(rec_ch ? f.y : f.x, y1, y2);
                        const float yb = FB(rec_ch ? f.w : f.z, ya, y1);
                        y2 = ya, y1 = yb;
                        rc[t] = ya, rc[t + 2] = yb;
                    }
                    if (t < hi_t) {
                        const float y = FB(rc[t], y1, y2);
                        y2 = y1, y1 = y;
                        rc[t] = y;
                    }
                }
                kb = kb + 1 == NBUF ? 0 : kb + 1;
                kh = kh + 1 == NHT ? 0 : kh + 1;
            }
            HOT_BAR();
        }
#undef FB
    } else if (mix_block >= 0) {
        // ---- stage C on tile it-2 (chain mode: wait for the CTA in front, add this CTA's rows to its running sum, hand it on) ----
        const uint32_t mix_t = ((uint32_t)mix_block * 32 + lane) * 4;
        uint32_t cb = 0, ch = 0;
        for (uint32_t it = 0; it < n_iter; it++) {
            if (it >= 2) {
                if (!HOT_SKIP(4)) {
                    const uint64_t m0 = m_begin + (uint64_t)(it - 2) * TT;
                    const bool full = m0 >= f_lo && m0 + TT <= f_hi;
                    hot_mix4(tiles + cb * tile_sz + HOT_PAD, s_ht[ch], s_rows, G, a.n_post, mix_t, full, m0, a.mix_len, partial, CHAIN, carry_row,
                             tagged_row, a.epoch * (n_iter + 1u) + (it - 2) + 1u);
                }
                cb = cb + 1 == NBUF ? 0 : cb + 1;
                ch = ch + 1 == NHT ? 0 : ch + 1;
            }
            HOT_BAR();
        }
    } else if (slot >= 0) {
        // ---- stage A on tile it ----
        const int first = hot_first_row<CHAIN>(slot), second = hot_second_row<CHAIN>(slot);
        const bool has_first = first >= 0 && (uint32_t)first < G;
        const bool has_second = second >= 0 && (uint32_t)second < G;
        const FusedRow& rowA = s_rows[has_first ? first : 0];
        const FusedRow& rowB = s_rows[has_second ? second : 0];
        // (lane's first frame * from) divmod to: shared by both rows when they have the same rate pair
        const bool same_rate = rowA.uni.from == rowB.uni.from && rowA.uni.to == rowB.uni.to;
        uint32_t lane_q = 0, lane_r = 0;
        if (has_first) {
            const uint32_t p = lane * (uint32_t)(TT / 32 / C) * rowA.uni.from;
            lane_q = p / rowA.uni.to;
            lane_r = p - lane_q * rowA.uni.to;
        }
        float xtail0[2 * C], xtail1[2 * C];   // x at the last two frames of the previous tile, per owned row
#pragma unroll
        for (int j = 0; j < 2 * C; j++) xtail0[j] = xtail1[j] = 0.f;
        uint32_t kw = 0, kb = 0, kh = 0, phase = 0;   // tile it
        for (uint32_t it = 0; it < n_iter; it++) {
            if (it < n_tiles) {
                if (has_first && !HOT_SKIP(1)) {
                    HOT_MBAR_WAIT(&s_full[kw], phase);
                    float* tile = tiles + kb * tile_sz + HOT_PAD;
                    const float* win = wins + kw * win_sz;
                    const int b = has_second ? second : first;
                    const HotTile& ha = s_ht[kh][first];
                    const HotTile& hb = s_ht[kh][b];
                    const bool do_second = has_second && !HOT_SKIP(8);
                    const float* win_a = win + first * wstride;
                    const float* win_b = win + b * wstride;
                    float* row_a = tile + first * ROW_STRIDE;
                    float* row_b = tile + b * ROW_STRIDE;
                    bool solo = true;
                    if constexpr (C == 1) {
                        if (do_second && same_rate && ha.interior && hb.interior && ha.r0 == hb.r0) {   // warp-uniform
                            solo = !(nogain ? hot_stage_a_pair<true, HASB>(rowA, rowB, ha, hb, a.n_pre, a.n_mid, lane, lane_q, lane_r, xtail0, xtail1, win_a, win_b, row_a, row_b)
                                            : hot_stage_a_pair<false, HASB>(rowA, rowB, ha, hb, a.n_pre, a.n_mid, lane, lane_q, lane_r, xtail0, xtail1, win_a, win_b, row_a, row_b));
                            HOT_PATH(solo ? HOT_PATH_PAIR_FAILED : HOT_PATH_PAIR, 2);
                        }
                    }
                    if (solo) {
                        if (ha.lo < ha.hi) {
                            if (nogain) hot_stage_a<true, C, HASB>(rowA, ha, a.n_pre, a.n_mid, lane, lane_q, lane_r, xtail0, win_a, row_a);
                            else hot_stage_a<false, C, HASB>(rowA, ha, a.n_pre, a.n_mid, lane, lane_q, lane_r, xtail0, win_a, row_a);
                        }
                        if (do_second && hb.lo < hb.hi) {
                            uint32_t qb = lane_q, rb = lane_r;
                            if (!same_rate) {
                                const uint32_t p = lane * (uint32_t)(TT / 32 / C) * rowB.uni.from;
                                qb = p / rowB.uni.to;
                                rb = p - qb * rowB.uni.to;
                            }
                            if (nogain) hot_stage_a<true, C, HASB>(rowB, hb, a.n_pre, a.n_mid, lane, qb, rb, xtail1, win_b, row_b);
                            else hot_stage_a<false, C, HASB>(rowB, hb, a.n_pre, a.n_mid, lane, qb, rb, xtail1, win_b, row_b);
                        }
                    }
                }
                kw = kw + 1 == NWIN ? 0 : kw + 1;
                phase ^= kw == 0;
                kb = kb + 1 == NBUF ? 0 : kb + 1;
                kh = kh + 1 == NHT ? 0 : kh + 1;
            }
            HOT_BAR();
        }
    } else {
        for (uint32_t it = 0; it < n_iter; it++) HOT_BAR();
    }
    HOT_TIMING_END
}

// ordered sum of the per-CTA partial rows
__global__ void __launch_bounds__(256) k_sum_partials(const float* __restrict__ partial, uint32_t n_ctas,
                                                      uint64_t mix_len, float* __restrict__ out) {
    for (uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; m < mix_len;
         m += (uint64_t)gridDim.x * blockDim.x) {
        float acc = partial[m];
        for (uint32_t c = 1; c < n_ctas; c++) acc = add(acc, partial[(uint64_t)c * mix_len + m]);
        out[m] = acc;
    }
}

}  // namespace

// ----------------------------------------------------------------------------------------------------
// host side: shape detection and launch
// ----------------------------------------------------------------------------------------------------
struct rb_fused_plan {
    FusedArgs args{};
    FusedRow* d_rows = nullptr;
    float* d_partial = nullptr;
    float* d_out = nullptr;
    uint32_t n_ctas = 0;
    uint32_t n_rec_warps = 0;
    uint32_t grid_y = 1;
    size_t smem_bytes = 0;
    bool single_cta_direct = false;
    bool all_f32 = true;
    bool hot = false;
    size_t hot_smem = 0;
    bool chain = false;               // RB_MIX_EXACT_ORDER on k_fused_hot: sequential sum across the CTAs (FusedArgs::chain)
    uint32_t* d_flags = nullptr;      // the ticket counter
    uint32_t epoch = 0;
    rb_lanes_plan* lanes = nullptr;   // RB_FUSED_LANES: the lane-per-stream kernel serves the batch (rb_lanes.cu)
    rb_fx_plan* fx = nullptr;         // the effect-chain kernel serves the batch (rb_fx.cu)
};

cudaError_t rb_fused_try_create(const rb_fused_stream* streams, size_t n_streams, uint16_t mixer_channels, float* d_out,
                                uint64_t mix_len, uint32_t flags, int sm_count, cudaStream_t st, rb_fused_plan** out) {
    *out = nullptr;
    if (n_streams == 0 || mix_len == 0) return cudaSuccess;
    // RB_MIX_EXACT_ORDER: the general path, except for filter-free resample -> gain -> mix batches, which k_lerp_mix sums in
    // one sequential chain per timeline position -- the reference's order (see below)
    const bool exact_order = (flags & RB_MIX_EXACT_ORDER) != 0;
    {   // spatial / reverb / AGC chains have a kernel of their own (with RB_MIX_EXACT_ORDER: its chain form, or nothing)
        rb_fx_plan* fx = nullptr;
        cudaError_t e = rb_fx_try_create(streams, n_streams, mixer_channels, d_out, mix_len, flags, st, &fx);
        if (e != cudaSuccess) return e;
        if (fx) {
            auto plan = new rb_fused_plan;
            plan->fx = fx;
            *out = plan;
            return cudaSuccess;
        }
    }
    std::vector<FusedRow> rows(n_streams);
    uint32_t n_pre = 0, n_mid = 0, n_post = 0, has_u = 0, has_b = 0, front = 0;
    bool mixed_u = false;   // some rows lost an identity conversion: only the lane kernel may take such a batch
    if (!fused_parse_rows(streams, n_streams, mixer_channels, rows, n_pre, n_mid, n_post, has_u, has_b, mixed_u, front)) return cudaSuccess;
    // RB_MIX_EXACT_ORDER: filter-free mono chains -> k_lerp_mix in one group; chains with a filter -> k_fused_hot with the running sum
    // handed from CTA to CTA (below); everything else -> the general path
    // (filter-free batches from 1024 streams on take the chain as well: k_lerp_mix in ONE group is one CTA per tile of the timeline
    // walking every stream, several times slower than the chain at 4096 streams x 2 s)
    auto hot_capable = [&]() {     // the same test as below, before anything is planned
        const uint32_t C = mixer_channels;
        bool ok = (has_b || has_u) && (C == 1 || C == 2);
        for (size_t i = 0; i < n_streams && ok; i++) {
            const FusedRow& r = rows[i];
            const uint64_t qT = (uint64_t)(TT / C) * r.uni.from / r.uni.to;
            ok = streams[i].fmt == RB_FMT_F32 && r.c_in == C && r.n_in % C == 0 && r.out_len % C == 0 && r.mix_start % C == 0 &&
                 (r.mode == ROW_DIRECT || r.mode == ROW_PASS || (r.mode == ROW_LERP && 3 + (qT + 3) * C <= (uint64_t)WSTRIDE)) &&
                 (has_b || r.mode == ROW_LERP);
        }
        return ok;
    };
    const bool exact_chain = exact_order && !front && !mixed_u && !(flags & (RB_FUSED_LANES | RB_FUSED_DUO)) &&
                             (has_b || (has_u && n_streams >= 1024 && !getenv("RB_EXACT_LERPMIX"))) && hot_capable();
    if (exact_order && !exact_chain && (has_b || front || !has_u || mixer_channels != 1 || (flags & RB_FUSED_LANES))) return cudaSuccess;
    if (has_b && (uint32_t)mixer_channels * 1u > 32u) return cudaSuccess;

    // Plain mixer of f32 sources at the mixer's own rate/channels (BASELINE cfg2): nothing to fuse -- the ordered
    // mix kernel of the general path reads every source once with 16-byte loads and is bit-exact.
    {
        bool plain = !has_b && !has_u && n_pre == 0 && n_mid == 0 && n_post == 0;
        for (size_t i = 0; i < n_streams && plain; i++) plain = streams[i].fmt == RB_FMT_F32 && streams[i].n_nodes == 0;
        if (plain) return cudaSuccess;
    }
    auto plan = new rb_fused_plan;
    plan->all_f32 = true;
    for (size_t i = 0; i < n_streams; i++) plan->all_f32 = plan->all_f32 && streams[i].fmt == RB_FMT_F32;
    if (!exact_chain) {
        cudaError_t e = fused_lanes_hook(rows, n_streams, mixer_channels, plan->all_f32, n_pre, n_mid, n_post, has_u, has_b, front, flags, sm_count,
                                         d_out, mix_len, st, &plan->lanes);
        if (e != cudaSuccess) {
            delete plan;
            return e;
        }
        if (exact_order && (!plan->lanes || rb_lanes_kind(plan->lanes) != 6)) {   // only k_lerp_mix keeps the sequential order
            rb_lanes_destroy(plan->lanes);
            delete plan;
            return cudaSuccess;
        }
        if (plan->lanes) {
            *out = plan;
            return cudaSuccess;
        }
        if (mixed_u) {   // the other fused kernels keep their one-shape rule: general path, as before
            delete plan;
            return cudaSuccess;
        }
    }
    const uint32_t C = mixer_channels;
    plan->hot = (has_b || has_u) && plan->all_f32 && (C == 1 || C == 2);
    bool narrow = plan->hot && has_b && C == 1;   // every row interpolates with a window of <= WSTRIDE_NARROW floats
    for (size_t i = 0; i < n_streams && plan->hot; i++) {
        FusedRow& r = rows[i];
        // the HOT kernel counts the index state in frames: C interleaved channels share one (i0, r0)
        const uint64_t qT = (uint64_t)(TT / C) * r.uni.from / r.uni.to;
        const bool window_fits = 3 + (qT + 3) * C <= (uint64_t)WSTRIDE;
        narrow = narrow && r.mode == ROW_LERP && 3 + (qT + 3) * C <= (uint64_t)WSTRIDE_NARROW;
        const bool whole_frames = r.n_in % C == 0 && r.out_len % C == 0 && r.mix_start % C == 0;
        plan->hot = r.c_in == C && whole_frames &&
                    (r.mode == ROW_DIRECT || r.mode == ROW_PASS || (r.mode == ROW_LERP && window_fits));
        // without a filter only rows that really interpolate take the HOT pipeline (the time axis is parallel as
        // well there: small batches are spread over the machine in time slices, see grid_y below)
        if (!has_b) plan->hot = plan->hot && r.mode == ROW_LERP;
    }
    if (exact_chain && !plan->hot) {   // only the HOT kernel hands the running sum on
        delete plan;
        return cudaSuccess;
    }
    if (plan->hot && !has_b && n_post == 0) {
        // no filter: the gains behind the resampler are the last thing before the sum -- apply them in stage C
        // (same single rounding per gain, same place in the chain) and keep stage A on its gain-free fast path
        for (size_t i = 0; i < n_streams; i++) {
            FusedRow& r = rows[i];
            for (uint32_t k = 0; k < n_mid; k++) r.post[k] = r.mid[k], r.mid[k] = 0.0f;
        }
        n_post = n_mid, n_mid = 0;
    }
    if (plan->hot) {
        for (size_t i = 0; i < n_streams; i++) {
            FusedRow& r = rows[i];
            r.q32 = r.uni.from / r.uni.to;          // HOT rows: the per-frame step
            r.r32 = r.uni.from % r.uni.to;
            r.qT = (uint32_t)((uint64_t)(TT / C) * r.uni.from / r.uni.to);
            r.rT = (uint32_t)((uint64_t)(TT / C) * r.uni.from % r.uni.to);
        }
    }
    // rows per CTA: one balanced wave over the SMs (k CTAs per SM when the batch is large)
    uint32_t S = (uint32_t)n_streams;
    const uint32_t wstride = narrow ? WSTRIDE_NARROW : WSTRIDE;
    uint32_t max_g = plan->hot ? (C == 2 ? HOT_MAX_ROWS_STEREO : narrow ? HOT_MAX_ROWS_NARROW : HOT_MAX_ROWS) : MAX_G;
    if (has_b) {
        while (max_g > 1 && max_g * mixer_channels > 128) max_g--;   // at most 4 recurrence warps
    }
    uint32_t k = (S + (uint32_t)sm_count * max_g - 1) / ((uint32_t)sm_count * max_g);
    uint32_t G = (S + (uint32_t)sm_count * k - 1) / ((uint32_t)sm_count * k);
    if (plan->hot && !has_b && S > (uint32_t)sm_count) {
        // full CTAs (every stage-A warp has a row); the machine is filled along the time axis instead.
        // (Up to one stream per SM the rule above gives G = 1: the sum stays in the reference's sequential order.)
        const uint32_t nx = (S + max_g - 1) / max_g;
        G = (S + nx - 1) / nx;
    }
    if (G > max_g) G = max_g;
    if (G < 1) G = 1;
    uint32_t n_ctas = (S + G - 1) / G;
    plan->n_ctas = n_ctas;
    plan->n_rec_warps = has_b ? (G * mixer_channels + 31) / 32 : 0;
    plan->smem_bytes = (size_t)(has_b ? NBUF : 1) * MAX_G * ROW_STRIDE * sizeof(float);
    plan->d_out = d_out;

    cudaError_t e = cudaMalloc(&plan->d_rows, n_streams * sizeof(FusedRow));
    if (e == cudaSuccess) e = cudaMemcpyAsync(plan->d_rows, rows.data(), n_streams * sizeof(FusedRow), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    plan->single_cta_direct = (n_ctas == 1);
    plan->chain = exact_chain && !plan->single_cta_direct;
    if (e == cudaSuccess && plan->chain) e = cudaMalloc(&plan->d_flags, sizeof(uint32_t));   // the ticket counter
    if (e == cudaSuccess && plan->chain) e = cudaMemsetAsync(plan->d_flags, 0, sizeof(uint32_t), st);
    const size_t row_bytes = plan->chain ? sizeof(uint2) : sizeof(float);   // chain: (value, tag) pairs, tag 0 = never written
    if (e == cudaSuccess && !plan->single_cta_direct) e = cudaMalloc(&plan->d_partial, (size_t)n_ctas * mix_len * row_bytes);
    if (e == cudaSuccess && !plan->single_cta_direct) e = cudaMemsetAsync(plan->d_partial, 0, (size_t)n_ctas * mix_len * row_bytes, st);
    plan->hot_smem = ((size_t)NBUF * ROW_STRIDE + (size_t)NWIN * wstride) * G * sizeof(float);
    if (e == cudaSuccess && plan->hot) {
        const int hs = (int)plan->hot_smem;
        const bool ch = plan->chain;
        auto set = [&](auto kern) { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, hs); };
        e = C == 2 ? (has_b ? (ch ? set(k_fused_hot<2, true, true>) : set(k_fused_hot<2, true, false>))
                            : (ch ? set(k_fused_hot<2, false, true>) : set(k_fused_hot<2, false, false>)))
                   : (has_b ? (ch ? set(k_fused_hot<1, true, true>) : set(k_fused_hot<1, true, false>))
                            : (ch ? set(k_fused_hot<1, false, true>) : set(k_fused_hot<1, false, false>)));
    }
    if (e == cudaSuccess && has_b) {
        const int sb = (int)plan->smem_bytes;
        e = cudaFuncSetAttribute(k_fused_biquad<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, sb);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_fused_biquad<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, sb);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_fused_biquad<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, sb);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_fused_biquad<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, sb);
    }
    if (e != cudaSuccess) {
        rb_fused_destroy(plan);
        return e;
    }
    FusedArgs& a = plan->args;
    a.rows = plan->d_rows, a.n_rows = S, a.rows_per_cta = G, a.c_mix = mixer_channels;
    a.n_pre = n_pre, a.n_mid = n_mid, a.n_post = n_post, a.has_biquad = has_b;
    a.partial = plan->single_cta_direct ? d_out : plan->d_partial;
    a.mix_len = mix_len;
    a.direct = plan->single_cta_direct ? 1u : 0u;
    a.chain = plan->chain ? 1u : 0u, a.out = d_out, a.flags = plan->d_flags;
    a.win_stride = wstride;
    // no-biquad variant: spread the timeline of each CTA over blockIdx.y so small batches still fill the GPU
    uint64_t tiles = (mix_len + TT - 1) / TT;
    uint64_t want_y = ((uint64_t)sm_count * 8 + n_ctas - 1) / n_ctas;
    if (plan->hot) want_y = has_b ? 1 : std::min<uint64_t>(((uint64_t)sm_count + n_ctas - 1) / n_ctas, std::max<uint64_t>(1, tiles / 8));
    if (plan->chain) want_y = 1;   // the chain walks the whole timeline in every CTA
    plan->grid_y = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(std::min<uint64_t>(tiles, want_y), 65535));
    *out = plan;
    return cudaSuccess;
}

void rb_fused_inputs_changed(rb_fused_plan* p) {
    if (p && p->lanes) rb_lanes_inputs_changed(p->lanes);
}

cudaError_t rb_fused_run(rb_fused_plan* p, cudaStream_t st, bool skip_final_sum) {
    if (p->fx) return rb_fx_run(p->fx, st);
    if (p->lanes) return rb_lanes_run(p->lanes, st);
    if (p->chain) p->args.epoch = p->epoch++;     // tickets and tags of this render
    const FusedArgs& a = p->args;
    if (p->hot) {
        const dim3 gb(p->n_ctas), gn(p->n_ctas, p->grid_y);
        if (p->chain) {
            if (a.c_mix == 1) {
                if (a.has_biquad) k_fused_hot<1, true, true><<<gb, 1024, p->hot_smem, st>>>(a);
                else k_fused_hot<1, false, true><<<gn, 1024, p->hot_smem, st>>>(a);
            } else {
                if (a.has_biquad) k_fused_hot<2, true, true><<<gb, 1024, p->hot_smem, st>>>(a);
                else k_fused_hot<2, false, true><<<gn, 1024, p->hot_smem, st>>>(a);
            }
        } else if (a.c_mix == 1) {
            if (a.has_biquad) k_fused_hot<1, true, false><<<gb, 1024, p->hot_smem, st>>>(a);
            else k_fused_hot<1, false, false><<<gn, 1024, p->hot_smem, st>>>(a);
        } else {
            if (a.has_biquad) k_fused_hot<2, true, false><<<gb, 1024, p->hot_smem, st>>>(a);
            else k_fused_hot<2, false, false><<<gn, 1024, p->hot_smem, st>>>(a);
        }
    } else if (a.has_biquad) {
        const uint32_t threads = 512;
        const bool mono = a.c_mix == 1;
        if (p->all_f32 && mono) k_fused_biquad<true, 1><<<p->n_ctas, threads, p->smem_bytes, st>>>(a, p->n_rec_warps);
        else if (p->all_f32) k_fused_biquad<true, 0><<<p->n_ctas, threads, p->smem_bytes, st>>>(a, p->n_rec_warps);
        else if (mono) k_fused_biquad<false, 1><<<p->n_ctas, threads, p->smem_bytes, st>>>(a, p->n_rec_warps);
        else k_fused_biquad<false, 0><<<p->n_ctas, threads, p->smem_bytes, st>>>(a, p->n_rec_warps);
    } else {
        if (p->all_f32) k_fused_nobiquad<true><<<dim3(p->n_ctas, p->grid_y), 256, p->smem_bytes, st>>>(a);
        else k_fused_nobiquad<false><<<dim3(p->n_ctas, p->grid_y), 256, p->smem_bytes, st>>>(a);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (!p->single_cta_direct && !p->chain && !skip_final_sum) {
        uint64_t blocks = (a.mix_len + 255) / 256;
        if (blocks > 132ull * 8) blocks = 132ull * 8;
        k_sum_partials<<<(uint32_t)blocks, 256, 0, st>>>(p->d_partial, p->n_ctas, a.mix_len, p->d_out);
        e = cudaGetLastError();
    }
    return e;
}

void rb_fused_destroy(rb_fused_plan* p) {
    if (!p) return;
    rb_lanes_destroy(p->lanes);
    rb_fx_destroy(p->fx);
    cudaFree(p->d_rows);
    cudaFree(p->d_partial);
    cudaFree(p->d_flags);
    delete p;
}

bool rb_fused_partial_rows(const rb_fused_plan* p, const float** partial, uint32_t* n_rows, uint64_t* pstride) {
    if (!p || p->fx || p->lanes || p->single_cta_direct || p->chain || !p->d_partial) return false;
    *partial = p->d_partial, *n_rows = p->n_ctas, *pstride = p->args.mix_len;
    return true;
}
uint32_t rb_fused_launch_count(const rb_fused_plan* p) {
    if (p->fx) return rb_fx_chain(p->fx) ? 1u : 2u;
    if (p->lanes) return rb_lanes_launch_count(p->lanes);
    return (p->single_cta_direct || p->chain) ? 1u : 2u;
}
int rb_fused_kind(const rb_fused_plan* p) { return p->fx ? 5 : p->lanes ? rb_lanes_kind(p->lanes) : (p->hot ? 1 : 0); }
uint32_t rb_fused_mix_group(const rb_fused_plan* p) {
    return p->fx ? (rb_fx_chain(p->fx) ? 0u : 4u) : p->lanes ? rb_lanes_mix_group(p->lanes) : p->chain ? 0u : p->args.rows_per_cta;   // chain: one sequential sum
}

#ifdef RB_HOT_TIMING
extern "C" int rb_debug_hot_skip(int mask) { return (int)cudaMemcpyToSymbol(g_hot_skip, &mask, sizeof(int)); }
extern "C" int rb_debug_hot_timing(unsigned long long* out, int reset) {
    cudaError_t e = cudaMemcpyFromSymbol(out, g_hot_timing, sizeof(unsigned long long) * 128);
    if (e == cudaSuccess && reset) {
        unsigned long long z[128] = {0};
        e = cudaMemcpyToSymbol(g_hot_timing, z, sizeof(z));
    }
    return (int)e;
}
#endif
#ifdef RB_HOT_PATHS
// out[HOT_PATH_*]: k_fused_hot's row-tiles per stage-A outcome since the last reset (8 counters, 5 in use)
extern "C" int rb_debug_hot_paths(unsigned long long* out, int reset) {
    cudaError_t e = cudaMemcpyFromSymbol(out, g_hot_paths, sizeof(unsigned long long) * HOT_PATH_N);
    if (e == cudaSuccess && reset) {
        unsigned long long z[HOT_PATH_N] = {0};
        e = cudaMemcpyToSymbol(g_hot_paths, z, sizeof(z));
    }
    return (int)e;
}
#endif
