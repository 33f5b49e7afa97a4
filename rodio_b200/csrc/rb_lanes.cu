// rb_lanes.cu — k_fused_lanes: the lane-per-stream fused kernel for large uniform batches (the warp program lives in
// rb_lanes_core.h, shared with the CPU emulator of tests/emu/), its input classification, the ordered sum of the
// per-warp partial rows, the FIFO kernels of the sessions, and the launchers; the host-side plan of a whole batch is
// rb_lanes_batch.cu (no device syntax there, so that the CPU suite can run it).
// Chosen by the fused planner for very large batches or on RB_FUSED_LANES (include/rodio_b200.h); also renders the blocks
// of the streaming sessions (rb_session_* in rb_api.cu).
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "rb_lanes.h"
#include "rb_lanes_plan.h"
#include "rb_duo_core.h"
#include "rb_dsp.cuh"

namespace {

constexpr int LANES_WARPS = 2;                      // warps per CTA: every warp is independent, small CTAs pack the SM
constexpr int LANES_THREADS = 32 * LANES_WARPS;
template <int C, bool DOWN>
constexpr int lanes_rs() { return lanes::Geo<C, DOWN ? lanes::NSLOT_DOWN : RB_LANES_UP_SLOTS>::RS; }
template <int C, bool DOWN>
constexpr size_t lanes_smem_bytes() { return (size_t)LANES_WARPS * 32 * lanes_rs<C, DOWN>() * sizeof(float); }   // 21.0 KB

template <int CI, int CO, bool HASB, bool FF2, int NPOST, bool PASS, bool PRE, bool FRONT, bool DOWN, bool GUARD, bool RESTART = false>
__global__ void __launch_bounds__(LANES_THREADS) k_fused_lanes(lanes::Args a) {
    extern __shared__ __align__(16) float lanes_smem[];
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t group = blockIdx.x * LANES_WARPS + warp;
    if (group >= a.n_groups) return;   // whole warps leave: the warp program only synchronises within a warp
    lanes::warp_main<CI, CO, HASB, FF2, NPOST, PASS, PRE, FRONT, DOWN, GUARD, RESTART>(a, group, lanes_smem + (size_t)warp * 32 * lanes::Geo<CI, DOWN ? lanes::NSLOT_DOWN : RB_LANES_UP_SLOTS>::RS);
}

// The lane-pair kernel (rb_duo_core.h): a warp = 64 mono streams, two per lane sharing one index state.
#ifndef RB_DUO_WARPS
#define RB_DUO_WARPS 1
#endif
constexpr int DUO_WARPS = RB_DUO_WARPS;   // every warp is independent; one per CTA balances 6.9 warps per SM (65 536 streams) as 7 : 6, not 8 : 6
constexpr size_t DUO_SMEM = (size_t)DUO_WARPS * duo::WARP_WORDS * sizeof(float);   // 17.0 KB
template <bool HASB, bool FF2, int NPOST>
__global__ void __launch_bounds__(32 * DUO_WARPS) k_fused_duo(lanes::Args a) {
    extern __shared__ __align__(16) float lanes_smem[];
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t group = blockIdx.x * DUO_WARPS + warp;
    if (group >= a.n_groups) return;
    duo::warp_main<HASB, FF2, NPOST>(a, group, lanes_smem + (size_t)warp * duo::WARP_WORDS);
}

// The same program on a PAIR of warps per group (rb_duo_core.h, ROLE): warp 0 feeds, warp 1 filters and sums.
constexpr size_t DUO_SPLIT_SMEM = (size_t)duo::WARP_WORDS * sizeof(float) + 2 * lanes::TILE * 32 * sizeof(simt::f2);   // 17.0 + 4 KB
template <bool HASB, bool FF2, int NPOST>
__global__ void __launch_bounds__(64) k_fused_duo_split(lanes::Args a) {
    extern __shared__ __align__(16) float lanes_smem[];
    const uint32_t group = blockIdx.x;
    if (group >= a.n_groups) return;
    simt::f2* handoff = reinterpret_cast<simt::f2*>(lanes_smem + duo::WARP_WORDS);
    if ((threadIdx.x >> 5) == 0) duo::warp_main<HASB, FF2, NPOST, 1>(a, group, lanes_smem, handoff);
    else duo::warp_main<HASB, FF2, NPOST, 2>(a, group, lanes_smem, handoff);
}

// ---------------------------------------------------------------------------------------------------
// k_lerp_mix: see rb_lanes.h.  256 threads, LM_U positions per thread (position = tile * 256 * LM_U + u * 256 + thread: consecutive
// lanes read consecutive input frames), grid (time tiles, stream groups).
// Arithmetic per sample: a + ((b - a) * num) / den with the division as the exact reciprocal step of the lane kernels for streams
// whose inputs are inside the class (k_classify_inputs), __fdiv_rn otherwise; (-0) / den keeps its sign.
// ---------------------------------------------------------------------------------------------------
constexpr int LM_U = 4;          // positions per thread: a tile is 256 * LM_U = 1024 timeline frames
constexpr int LM_ROWS = 4;       // rows per pipeline stage (50 KB of windows per CTA: four CTAs per SM)
constexpr int LM_STAGES = 3;     // stages in shared memory: one being summed, two in flight
constexpr int LM_GROUP = 64;     // row descriptors staged at a time (= the largest group the planner makes)
constexpr int LM_WQ = 260;       // 16-byte quads of one row's window: 1024 * from / to + 2 frames (from < to) + alignment slack
constexpr uint32_t LM_SMEM = LM_STAGES * LM_ROWS * LM_WQ * 16;
__device__ __forceinline__ void lm_cp16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void lm_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void lm_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// The input window of a (row, tile) -- the frames [i_tile, i_tile + n_win) of the row, 1024 * 147 / 160 + 2 of them at 44.1 -> 48 kHz --
// travels HBM -> shared memory by 16-byte cp.async (SASS LDGSTS.E.BYPASS.128), LM_ROWS rows per stage and two stages ahead of the
// sums: the copies of 16 rows are in flight while 8 are summed, whatever order the compiler gives the arithmetic (the first
// version left every load to LDG.32 pairs in front of their use and stalled on long scoreboards).  Rows that do not interpolate on the whole tile (a stream starts or ends inside it) or whose inputs are outside
// the exact-reciprocal class skip the window and read global memory directly, with the IEEE division.
struct LmSlot {       // what the summing loop needs of a row: 8 bytes, one LDS.64
    float post;       // the one gain (1.0: none)
    uint32_t woff;    // float offset of the row's first frame inside its stage buffer; LM_GLOBAL: the row reads global memory
};
constexpr uint32_t LM_GLOBAL = 0xffffffffu;
template <int NPOST>
__global__ void __launch_bounds__(256) k_lerp_mix(rb_lerpmix_args a) {
    extern __shared__ __align__(16) unsigned char lm_smem[];
    __shared__ rb_lerpmix_row s_rows[LM_GROUP];
    __shared__ LmSlot s_slot[LM_GROUP];
    float4* const win = reinterpret_cast<float4*>(lm_smem);
    const uint64_t tile_lo = (uint64_t)blockIdx.x * (256 * LM_U);
    if (tile_lo >= a.mix_len) return;
    const uint64_t tile_hi = min(a.mix_len, tile_lo + 256 * LM_U);
    const uint32_t g = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t r_lo = g * a.rows_per_group, r_hi = min(a.n_rows, r_lo + a.rows_per_group);
    uint32_t tap[LM_U], pos[LM_U];     // tap: left input frame of the position, relative to the tile's first
    float numf[LM_U], acc[LM_U];
    bool any[LM_U];
    // origin <= every position that any stream covers, and origin need not be a multiple of the tile: the tile's taps start at
    // base, and a position in front of it (no stream covers it) takes base's tap, so that no subtraction below wraps around
    const uint64_t base = max(tile_lo, a.origin);
    const uint64_t i_tile = ((base - a.origin) * (uint64_t)a.from) / a.to;
    const uint32_t n_win = (uint32_t)((((max(tile_hi - 1, base) - a.origin) * (uint64_t)a.from) / a.to) - i_tile) + 2;   // frames a full row needs
#pragma unroll
    for (int u = 0; u < LM_U; u++) {
        const uint64_t n = tile_lo + (uint64_t)u * 256 + threadIdx.x;
        const uint64_t prod = (max(n, base) - a.origin) * (uint64_t)a.from;
        const uint64_t i = prod / a.to;
        tap[u] = (uint32_t)(i - i_tile), numf[u] = __uint2float_rn((uint32_t)(prod - i * a.to)), pos[u] = (uint32_t)n;
        acc[u] = 0.0f, any[u] = false;
    }
    const float den = a.den_f, rcp = a.rcp_den;
    const uint32_t t_lo = (uint32_t)tile_lo, t_hi = (uint32_t)tile_hi;
    const bool win_ok = n_win + 3 <= LM_WQ * 4;   // the planner only sends from < to here; anything else reads global memory
    const bool full_tile = tile_hi - tile_lo == 256 * LM_U;
    bool any_win = false;                          // a window row covers every position of the tile
    for (uint32_t rs = r_lo; rs < r_hi; rs += LM_GROUP) {
        const uint32_t n_st = min((uint32_t)LM_GROUP, r_hi - rs);
        __syncthreads();               // the previous group's descriptors and windows are no longer read
        if (threadIdx.x < n_st) {
            const rb_lerpmix_row row = a.rows[rs + threadIdx.x];
            const bool unsafe = (a.lane_rows[row.row].flags & lanes::ROW_UNSAFE) != 0;
            // the window path: the row interpolates on the whole tile and its inputs are inside the exact-reciprocal class
            const bool w_ok = win_ok && !unsafe && row.lo <= t_lo && row.hi_int >= t_hi;
            const uint32_t off = (uint32_t)((reinterpret_cast<uintptr_t>(row.p + i_tile) >> 2) & 3u);
            s_rows[threadIdx.x] = row;
            s_slot[threadIdx.x] = LmSlot{row.post, w_ok ? (threadIdx.x % LM_ROWS) * (LM_WQ * 4) + off : LM_GLOBAL};
        }
        __syncthreads();
        const uint32_t n_stages = (n_st + LM_ROWS - 1) / LM_ROWS;
        auto issue = [&](uint32_t stage) {          // warps 2j and 2j + 1 copy row j of the stage: 16 bytes per lane and step
            const uint32_t jrow = warp >> 1;
            const uint32_t r = stage * LM_ROWS + jrow;
            if (stage < n_stages && r < n_st) {
                const uint32_t woff = s_slot[r].woff;
                if (woff != LM_GLOBAL) {
                    const uint32_t off = woff & 3u;
                    const float4* src4 = reinterpret_cast<const float4*>(s_rows[r].p + i_tile - off);
                    float4* dst4 = win + (size_t)(stage % LM_STAGES) * LM_ROWS * LM_WQ + jrow * LM_WQ;
                    const uint32_t nq = (off + n_win + 3) >> 2;
                    for (uint32_t q = lane + 32 * (warp & 1); q < nq; q += 64) lm_cp16(dst4 + q, src4 + q);
                }
            }
            lm_commit();               // an empty group keeps the wait counts uniform
        };
        issue(0);
        issue(1);
        for (uint32_t stage = 0; stage < n_stages; stage++) {
            lm_wait<1>();              // this thread's copies of `stage` have landed ...
            __syncthreads();           // ... and everybody else's; everybody is also done reading stage - 1
            issue(stage + 2);          // into the buffer of stage - 1
            const float* buf = reinterpret_cast<const float*>(win + (size_t)(stage % LM_STAGES) * LM_ROWS * LM_WQ);
            const uint32_t j_hi = min((uint32_t)LM_ROWS, n_st - stage * LM_ROWS);
            for (uint32_t j = 0; j < j_hi; j++) {
                const LmSlot sl = s_slot[stage * LM_ROWS + j];
                if (sl.woff != LM_GLOBAL) {
                    const float* __restrict__ w = buf + sl.woff;
                    float xa[LM_U], xb[LM_U];
#pragma unroll
                    for (int u = 0; u < LM_U; u++) xa[u] = w[tap[u]], xb[u] = w[tap[u] + 1];
#pragma unroll
                    for (int u = 0; u < LM_U; u++) {
                        // a + ((b - a) * num) / den with the division as the exact reciprocal step; m = -0 gives q = +0 here where the
                        // division gives -0: x can then differ in the sign of a zero only, which a sum that starts from +0.0 cannot see
                        const float m = __fmul_rn(__fsub_rn(xb[u], xa[u]), numf[u]);
                        const float q0 = __fmul_rn(m, rcp);
                        const float q = __fmaf_rn(__fmaf_rn(-q0, den, m), rcp, q0);
                        float x = __fadd_rn(xa[u], q);
                        if (NPOST) x = __fmul_rn(x, sl.post);
                        if (full_tile || pos[u] < t_hi) acc[u] = __fadd_rn(acc[u], x);      // the last tile of the timeline may be partial
                    }
                    any_win = true;
                    continue;
                }
                const rb_lerpmix_row row = s_rows[stage * LM_ROWS + j];
                if (row.hi <= t_lo || row.lo >= t_hi) continue;          // the stream is silent on this tile
                const float* __restrict__ p = row.p + i_tile;
#pragma unroll
                for (int u = 0; u < LM_U; u++) {
                    if (pos[u] < row.lo || pos[u] >= row.hi || pos[u] >= t_hi) continue;
                    const float xa = __ldg(p + tap[u]);
                    float x = xa;
                    if (pos[u] < row.hi_int) x = __fadd_rn(xa, __fdiv_rn(__fmul_rn(__fsub_rn(__ldg(p + tap[u] + 1), xa), numf[u]), den));
                    if (NPOST) x = __fmul_rn(x, row.post);
                    acc[u] = __fadd_rn(acc[u], x), any[u] = true;
                }
            }
        }
        lm_wait<0>();
    }
    float* __restrict__ out = a.out + (uint64_t)g * a.pstride;
#pragma unroll
    for (int u = 0; u < LM_U; u++)
        if (pos[u] < t_hi && (any[u] || any_win || a.n_groups == 1)) out[pos[u]] = acc[u];
}

// One CTA per stream: does every non-zero |x| lie inside [2^-70, 2^60]?  (rb_lanes_core.h, "Exact division".)
// channels[r]: interleaved channels of stream r.
__global__ void __launch_bounds__(256) k_classify_inputs(lanes::Row* rows, uint32_t n_rows, const uint8_t* __restrict__ channels) {
    const uint32_t r = blockIdx.x;
    if (r >= n_rows) return;
    const float* __restrict__ x = rows[r].in;
    const uint64_t L = rows[r].L * channels[r];   // floats
    bool bad = false;
    const uint64_t n4 = L / 4;
    const float4* __restrict__ x4 = reinterpret_cast<const float4*>(x);
    auto out_of_class = [](float v) {
        const uint32_t u = __float_as_uint(v) & 0x7fffffffu;
        return u != 0u && (u - 0x1c800000u) >= (0x5d800000u - 0x1c800000u);
    };
    for (uint64_t i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = __ldg(x4 + i);
        bad |= out_of_class(v.x) | out_of_class(v.y) | out_of_class(v.z) | out_of_class(v.w);
    }
    for (uint64_t i = n4 * 4 + threadIdx.x; i < L; i += blockDim.x) bad |= out_of_class(__ldg(x + i));
    const int any = __syncthreads_or(bad ? 1 : 0);
    if (threadIdx.x == 0) rows[r].flags = (rows[r].flags & ~lanes::ROW_UNSAFE) | (any ? lanes::ROW_UNSAFE : 0u);
}

__global__ void __launch_bounds__(256) k_spread_flags(lanes::Row* rows, uint32_t n_rows, const uint32_t* __restrict__ row_stream,
                                                      const lanes::Row* __restrict__ stream_rows) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const uint32_t s = row_stream[r];
    const uint32_t bad = s == ~0u ? 0u : (stream_rows[s].flags & lanes::ROW_UNSAFE);
    rows[r].flags = (rows[r].flags & ~lanes::ROW_UNSAFE) | bad;
}

// out[m] = +0.0 + partial[0][m] + partial[1][m] + ...  (warp order = insertion order of the streams)
__global__ void __launch_bounds__(256) k_sum_groups(const float* __restrict__ partial, uint32_t n_groups, uint64_t pstride,
                                                    uint64_t mix_len, float* __restrict__ out) {
    for (uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; m < mix_len; m += (uint64_t)gridDim.x * blockDim.x) {
        float acc = 0.0f;
        for (uint32_t g = 0; g < n_groups; g++) acc = __fadd_rn(acc, partial[(uint64_t)g * pstride + m]);
        out[m] = acc;
    }
}

// out[f * C + j] = +0.0 + partial[g][f * w + j - o] for every group g (in order) whose slot [o, o + w) covers mixer channel j
__global__ void __launch_bounds__(256) k_sum_slots(const float* __restrict__ partial, const uint32_t* __restrict__ slot, uint32_t n_groups,
                                                   uint64_t pstride, uint64_t n_floats, uint32_t channels, float* __restrict__ out) {
    for (uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; m < n_floats; m += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t f = m / channels;
        const uint32_t j = (uint32_t)(m - f * channels);
        float acc = 0.0f;
        for (uint32_t g = 0; g < n_groups; g++) {
            const uint32_t s = __ldg(slot + g), c = j - (s & 0xffffu), w = s >> 16;
            if (c < w) acc = __fadd_rn(acc, partial[(uint64_t)g * pstride + f * w + c]);
        }
        out[m] = acc;
    }
}

// A push program on sample n of its source (rb_lanes.h: rb_prog_op), in chain order.  Past a take's count the sample is the
// take's Sample::EQUILIBRIUM padding, which the ops behind it still see.
__device__ __forceinline__ float run_prog(float v, uint64_t n, uint32_t C, const rb_prog_op* __restrict__ ops, uint32_t n_ops) {
    for (uint32_t k = 0; k < n_ops; k++) {
        const rb_prog_op& op = ops[k];
        switch (op.kind) {
            case RB_N_AMPLIFY: v = rbd::mul(v, op.p.amp); break;
            case RB_N_DISTORT: v = rbd::distort_sample(v, op.p.dist.gain, op.p.dist.threshold); break;
            case RB_N_RAMP: {
                const rb_ramp_params& r = op.p.ramp;
                const float factor = rbd::ramp_factor((n / C) * r.dt_ns, r.total_ns, r.start, r.end, r.clamp_end ? r.end : 1.0f,
                                                      rbd::duration_secs_f32(r.total_ns));
                v = rbd::mul(v, factor);
                break;
            }
            default: {   // RB_N_TAKE
                const rb_take_params& t = op.p.take;
                if (n < t.count) {
                    if (t.fadeout) v = rbd::take_fade(v, n, t.total_ns, t.dps_ns, t.total_ms_f);
                } else {
                    v = 0.0f;
                }
            }
        }
    }
    return v;
}

// FIFO scatter + sticky classification, one CTA per job (rb_lanes.h).  PROG: the jobs are rb_fifo_prog_job and every sample
// runs through its source's push program first.
template <bool PROG>
__global__ void __launch_bounds__(128) k_fifo_scatter(const float* __restrict__ staging, const void* __restrict__ jobs_,
                                                      float* __restrict__ fifo, uint64_t stride, uint32_t* __restrict__ flags,
                                                      const rb_prog_op* __restrict__ ops) {
    const rb_fifo_job j = PROG ? static_cast<const rb_fifo_prog_job*>(jobs_)[blockIdx.x].j : static_cast<const rb_fifo_job*>(jobs_)[blockIdx.x];
    const uint32_t ci = j.ci, n = j.frames * ci;
    const float* __restrict__ src = staging + j.src + j.ch0;
    float* __restrict__ dst = fifo + (uint64_t)j.row * stride + (uint64_t)j.fill * ci;
    uint64_t base = 0;
    uint32_t op0 = 0, n_ops = 0;
    if (PROG) {
        const rb_fifo_prog_job& pj = static_cast<const rb_fifo_prog_job*>(jobs_)[blockIdx.x];
        base = pj.base, op0 = pj.op0, n_ops = pj.n_ops;
    }
    bool bad = false;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t f = ci == 1 ? i : i >> 1;
        float v = src[(uint64_t)f * j.src_ch + (i - f * ci)];
        if (PROG) v = run_prog(v, (base + f) * j.src_ch + j.ch0 + (i - f * ci), j.src_ch, ops + op0, n_ops);
        const uint32_t u = __float_as_uint(v) & 0x7fffffffu;
        bad |= u != 0u && (u - 0x1c800000u) >= (0x5d800000u - 0x1c800000u);
        dst[i] = v;
    }
    if (__syncthreads_or(bad ? 1 : 0) && threadIdx.x == 0) flags[j.row] = 1u;
}

// Generator fill (rb_lanes.h: rb_fifo_gen_job), k_siggen's shape (rb_kernels.cu): GEN_PER_CTA generators per CTA.  The phase is a
// serial f32 recurrence that drifts by design (signal_generator.rs:133), so warp 0, lane = generator, walks exactly `frames` steps of
// it a tile ahead into shared memory; the seven other warps evaluate the waveform of the previous tile, run the program, classify
// and store with consecutive threads on consecutive samples.
constexpr int GEN_TILE = 256, GEN_THREADS = 256, GEN_PITCH = GEN_TILE + 1, GEN_PER_CTA = 4;
__global__ void __launch_bounds__(GEN_THREADS) k_fifo_generate(const rb_fifo_gen_job* __restrict__ jobs, uint32_t n_jobs,
                                                               const rb_prog_op* __restrict__ ops, const float* __restrict__ phase_in,
                                                               float* __restrict__ phase_out, float* __restrict__ fifo, uint64_t stride,
                                                               uint32_t* __restrict__ flags) {
    __shared__ float s_phase[2][GEN_PER_CTA * GEN_PITCH];
    __shared__ rb_fifo_gen_job s_job[GEN_PER_CTA];
    __shared__ uint32_t s_bad;
    const uint32_t j0 = blockIdx.x * GEN_PER_CTA, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n_g = min((uint32_t)GEN_PER_CTA, n_jobs - j0);
    if (threadIdx.x < n_g) s_job[threadIdx.x] = jobs[j0 + threadIdx.x];
    if (threadIdx.x == 0) s_bad = 0;
    __syncthreads();
    uint32_t max_n = 0;
    for (uint32_t g = 0; g < n_g; g++) max_n = max(max_n, s_job[g].frames);
    const uint32_t n_tiles = (max_n + GEN_TILE - 1) / GEN_TILE;
    float phase = 0.0f;
    if (warp == 0 && lane < n_g) phase = phase_in[s_job[lane].gen];
    uint32_t bad = 0;   // worker threads: bit g = a sample of generator g lies outside the exact-reciprocal class
    for (uint32_t it = 0; it <= n_tiles; it++) {
        if (warp == 0) {
            const uint32_t lo = it * GEN_TILE;
            if (it < n_tiles && lane < n_g && lo < s_job[lane].frames) {
                float* row = &s_phase[it & 1][lane * GEN_PITCH];
                const uint32_t cnt = min((uint32_t)GEN_TILE, s_job[lane].frames - lo);
                const float step = s_job[lane].step;
                if (step < 1.0f) {
#pragma unroll 8
                    for (uint32_t t = 0; t < cnt; t++) row[t] = phase, phase = rbd::signal_phase_next<true>(phase, step);
                } else {
                    for (uint32_t t = 0; t < cnt; t++) row[t] = phase, phase = rbd::signal_phase_next<false>(phase, step);
                }
            }
        } else if (it > 0) {
            const uint32_t lo = (it - 1) * GEN_TILE;
            for (uint32_t w = threadIdx.x - 32; w < n_g * GEN_TILE; w += GEN_THREADS - 32) {
                const uint32_t g = w / GEN_TILE, t = w % GEN_TILE;
                const rb_fifo_gen_job& j = s_job[g];
                if (lo + t >= j.frames) continue;
                float v = rbd::signal_value(j.fn, s_phase[(it - 1) & 1][g * GEN_PITCH + t]);
                v = run_prog(v, j.base + lo + t, 1, ops + j.op0, j.n_ops);
                const uint32_t u = __float_as_uint(v) & 0x7fffffffu;
                if (u != 0u && (u - 0x1c800000u) >= (0x5d800000u - 0x1c800000u)) bad |= 1u << g;
                fifo[(uint64_t)j.row * stride + j.fill + lo + t] = v;
            }
        }
        __syncthreads();
    }
    if (bad) atomicOr(&s_bad, bad);
    if (warp == 0 && lane < n_g) phase_out[s_job[lane].gen] = phase;
    __syncthreads();
    if (threadIdx.x < n_g && ((s_bad >> threadIdx.x) & 1u)) flags[s_job[threadIdx.x].row] = 1u;
}

__global__ void __launch_bounds__(128) k_fifo_compact(const float* __restrict__ src, float* __restrict__ dst, uint64_t stride,
                                                      const uint32_t* __restrict__ drop, const uint32_t* __restrict__ keep) {
    const uint32_t r = blockIdx.x, n = keep[r];
    const float* __restrict__ s = src + (uint64_t)r * stride + drop[r];   // drop is a multiple of 4: both sides 16-byte aligned
    float* __restrict__ d = dst + (uint64_t)r * stride;
    const uint32_t n4 = n / 4;
    for (uint32_t i = threadIdx.x; i < n4; i += blockDim.x)
        reinterpret_cast<float4*>(d)[i] = reinterpret_cast<const float4*>(s)[i];
    for (uint32_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
}

template <int CI, int CO, bool HASB, bool FF2, int NPOST, bool PASS, bool PRE, bool FRONT = false, bool DOWN = false, bool GUARD = false>
static void launch_lanes(const lanes::Args& a, cudaStream_t st) {
    const uint32_t n_ctas = (a.n_groups + LANES_WARPS - 1) / LANES_WARPS;
    k_fused_lanes<CI, CO, HASB, FF2, NPOST, PASS, PRE, FRONT, DOWN, GUARD><<<n_ctas, LANES_THREADS, lanes_smem_bytes<CI, DOWN>(), st>>>(a);   // < 48 KB: no opt-in needed
}
template <int CI, int CO, bool PASS, bool PRE, bool GUARD = false>
static void launch_lanes_c(const lanes::Args& a, bool has_biquad, bool ff2, bool has_post, cudaStream_t st) {
    if (has_biquad) {
        if (ff2) has_post ? launch_lanes<CI, CO, true, true, 1, PASS, PRE, false, false, GUARD>(a, st) : launch_lanes<CI, CO, true, true, 0, PASS, PRE, false, false, GUARD>(a, st);
        else has_post ? launch_lanes<CI, CO, true, false, 1, PASS, PRE, false, false, GUARD>(a, st) : launch_lanes<CI, CO, true, false, 0, PASS, PRE, false, false, GUARD>(a, st);
    } else {
        has_post ? launch_lanes<CI, CO, false, false, 1, PASS, PRE, false, false, GUARD>(a, st) : launch_lanes<CI, CO, false, false, 0, PASS, PRE, false, false, GUARD>(a, st);
    }
}
template <int CI, int CO>
static void launch_lanes_cc(const lanes::Args& a, bool has_biquad, bool ff2, bool has_post, bool has_pre, bool front, bool guard, cudaStream_t st) {
    const bool pass = a.from == a.to;   // sources at the mixer's rate: taps used raw
    if (front) {                        // the filter in front of the conversion: plain coefficients, Row::pre always applied
        if (lanes::ratio_runs_down(a.from, a.to))
            has_post ? launch_lanes<CI, CO, true, false, 1, false, false, true, true>(a, st) : launch_lanes<CI, CO, true, false, 0, false, false, true, true>(a, st);
        else if (pass) has_post ? launch_lanes<CI, CO, true, false, 1, true, false, true>(a, st) : launch_lanes<CI, CO, true, false, 0, true, false, true>(a, st);
        else has_post ? launch_lanes<CI, CO, true, false, 1, false, false, true>(a, st) : launch_lanes<CI, CO, true, false, 0, false, false, true>(a, st);
        return;
    }
    if (lanes::ratio_runs_down(a.from, a.to)) {   // above the mixer's rate, up to twice: fast tiles of their own, Row::pre always applied
        if (has_biquad) {
            if (ff2) has_post ? launch_lanes<CI, CO, true, true, 1, false, false, false, true>(a, st) : launch_lanes<CI, CO, true, true, 0, false, false, false, true>(a, st);
            else has_post ? launch_lanes<CI, CO, true, false, 1, false, false, false, true>(a, st) : launch_lanes<CI, CO, true, false, 0, false, false, false, true>(a, st);
        } else {
            has_post ? launch_lanes<CI, CO, false, false, 1, false, false, false, true>(a, st) : launch_lanes<CI, CO, false, false, 0, false, false, false, true>(a, st);
        }
        return;
    }
    if (pass) has_pre ? launch_lanes_c<CI, CO, true, true>(a, has_biquad, ff2, has_post, st) : launch_lanes_c<CI, CO, true, false>(a, has_biquad, ff2, has_post, st);
    else if (has_pre && guard) launch_lanes_c<CI, CO, false, true, true>(a, has_biquad, ff2, has_post, st);   // a gain in front out of range
    else has_pre ? launch_lanes_c<CI, CO, false, true>(a, has_biquad, ff2, has_post, st) : launch_lanes_c<CI, CO, false, false>(a, has_biquad, ff2, has_post, st);
}

// The RESTART twins (rb_lanes_core.h: Cut).  One per (layout, filter, FRONT, DOWN): the twin of an up-sampling class is the
// guarded PRE tile, and every twin takes plain coefficients and applies Row::post -- a gain of 1.0, the guard and the three-product
// feed-forward give the bits of the variants they stand in for, and a class only comes here for the blocks that hold a cut.
template <int CI, int CO>
static void launch_restart_cc(const lanes::Args& a, bool has_biquad, bool front, cudaStream_t st) {
    const uint32_t n_ctas = (a.n_groups + LANES_WARPS - 1) / LANES_WARPS;
    const bool down = lanes::ratio_runs_down(a.from, a.to);
#define RB_RESTART(HASB, PRE, FRONT, DOWN, GUARD) \
    k_fused_lanes<CI, CO, HASB, false, 1, false, PRE, FRONT, DOWN, GUARD, true><<<n_ctas, LANES_THREADS, lanes_smem_bytes<CI, DOWN>(), st>>>(a)
    if (front) down ? RB_RESTART(true, false, true, true, false) : RB_RESTART(true, false, true, false, false);
    else if (down) has_biquad ? RB_RESTART(true, false, false, true, false) : RB_RESTART(false, false, false, true, false);
    else has_biquad ? RB_RESTART(true, true, false, false, true) : RB_RESTART(false, true, false, false, true);
#undef RB_RESTART
}

}  // namespace

cudaError_t rb_lanes_launch_restart(const lanes::Args& a, uint32_t ch_in, uint32_t ch_out, bool has_biquad, bool front, cudaStream_t st) {
    if (a.mix_len == 0 || a.n_groups == 0) return cudaSuccess;
    if (!a.cuts || !a.cut_first || a.from == a.to || (front && !has_biquad)) return cudaErrorInvalidValue;
    if (!((ch_in == 1 || ch_in == 2) && (ch_in == ch_out || (ch_in == 1 && ch_out == 2)))) return cudaErrorInvalidValue;
    if (ch_in == 2) launch_restart_cc<2, 2>(a, has_biquad, front, st);
    else if (ch_out == 2) launch_restart_cc<1, 2>(a, has_biquad, front, st);
    else launch_restart_cc<1, 1>(a, has_biquad, front, st);
    return cudaGetLastError();
}

cudaError_t rb_lanes_launch_kernel(const lanes::Args& a, uint32_t ch_in, uint32_t ch_out, bool has_biquad, bool ff2, bool has_post,
                                   bool has_pre, bool front, bool guard, cudaStream_t st) {
    if (a.mix_len == 0 || a.n_groups == 0) return cudaSuccess;
    if (front && !has_biquad) return cudaErrorInvalidValue;
    if (!((ch_in == 1 || ch_in == 2) && (ch_in == ch_out || (ch_in == 1 && ch_out == 2)))) return cudaErrorInvalidValue;
    if (ch_in == 2) launch_lanes_cc<2, 2>(a, has_biquad, ff2, has_post, has_pre, front, guard, st);
    else if (ch_out == 2) launch_lanes_cc<1, 2>(a, has_biquad, ff2, has_post, has_pre, front, guard, st);
    else launch_lanes_cc<1, 1>(a, has_biquad, ff2, has_post, has_pre, front, guard, st);
    return cudaGetLastError();
}

// k_fused_duo over a.rows: a.n_groups counts groups of 64 rows
cudaError_t rb_duo_launch_kernel(const lanes::Args& a, bool has_biquad, bool ff2, bool has_post, cudaStream_t st) {
    if (a.mix_len == 0 || a.n_groups == 0) return cudaSuccess;
    static const bool split = []() { const char* e = getenv("RB_DUO_SPLIT"); return e ? atoi(e) != 0 : false; }();   // the split pair of warps, kept for A/B runs
    if (split) {
        const dim3 g(a.n_groups), b(64);
        if (has_biquad) {
            if (ff2) has_post ? k_fused_duo_split<true, true, 1><<<g, b, DUO_SPLIT_SMEM, st>>>(a) : k_fused_duo_split<true, true, 0><<<g, b, DUO_SPLIT_SMEM, st>>>(a);
            else has_post ? k_fused_duo_split<true, false, 1><<<g, b, DUO_SPLIT_SMEM, st>>>(a) : k_fused_duo_split<true, false, 0><<<g, b, DUO_SPLIT_SMEM, st>>>(a);
        } else {
            has_post ? k_fused_duo_split<false, false, 1><<<g, b, DUO_SPLIT_SMEM, st>>>(a) : k_fused_duo_split<false, false, 0><<<g, b, DUO_SPLIT_SMEM, st>>>(a);
        }
        return cudaGetLastError();
    }
    const uint32_t n_ctas = (a.n_groups + DUO_WARPS - 1) / DUO_WARPS;
    const dim3 g(n_ctas), b(32 * DUO_WARPS);
    if (has_biquad) {
        if (ff2) has_post ? k_fused_duo<true, true, 1><<<g, b, DUO_SMEM, st>>>(a) : k_fused_duo<true, true, 0><<<g, b, DUO_SMEM, st>>>(a);
        else has_post ? k_fused_duo<true, false, 1><<<g, b, DUO_SMEM, st>>>(a) : k_fused_duo<true, false, 0><<<g, b, DUO_SMEM, st>>>(a);
    } else {
        has_post ? k_fused_duo<false, false, 1><<<g, b, DUO_SMEM, st>>>(a) : k_fused_duo<false, false, 0><<<g, b, DUO_SMEM, st>>>(a);
    }
    return cudaGetLastError();
}

cudaError_t rb_lerpmix_launch(const rb_lerpmix_args& a, cudaStream_t st) {
    if (a.mix_len == 0 || a.n_rows == 0) return cudaSuccess;
    const dim3 grid((uint32_t)((a.mix_len + 256 * LM_U - 1) / (256 * LM_U)), a.n_groups);
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(k_lerp_mix<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LM_SMEM);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_lerp_mix<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LM_SMEM);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    if (a.has_post) k_lerp_mix<1><<<grid, 256, LM_SMEM, st>>>(a);
    else k_lerp_mix<0><<<grid, 256, LM_SMEM, st>>>(a);
    return cudaGetLastError();
}

cudaError_t rb_lanes_launch_sum(const float* d_partial, uint32_t n_groups, uint64_t pstride, uint64_t n_floats, float* d_out,
                                cudaStream_t st) {
    if (n_floats == 0) return cudaSuccess;
    uint64_t blocks = (n_floats + 255) / 256;
    if (blocks > 132ull * 8) blocks = 132ull * 8;
    k_sum_groups<<<(uint32_t)blocks, 256, 0, st>>>(d_partial, n_groups, pstride, n_floats, d_out);
    return cudaGetLastError();
}

cudaError_t rb_lanes_launch_sum_slots(const float* d_partial, const uint32_t* d_slot, uint32_t n_groups, uint64_t pstride, uint64_t n_frames,
                                      uint32_t channels, float* d_out, cudaStream_t st) {
    const uint64_t n_floats = n_frames * channels;
    if (n_floats == 0) return cudaSuccess;
    uint64_t blocks = (n_floats + 255) / 256;
    if (blocks > 132ull * 8) blocks = 132ull * 8;
    k_sum_slots<<<(uint32_t)blocks, 256, 0, st>>>(d_partial, d_slot, n_groups, pstride, n_floats, channels, d_out);
    return cudaGetLastError();
}

cudaError_t rb_lanes_fifo_scatter(const float* d_staging, const rb_fifo_job* d_jobs, uint32_t n_jobs, float* d_fifo, uint64_t stride,
                                  uint32_t* d_flags, cudaStream_t st) {
    if (n_jobs == 0) return cudaSuccess;
    k_fifo_scatter<false><<<n_jobs, 128, 0, st>>>(d_staging, d_jobs, d_fifo, stride, d_flags, nullptr);
    return cudaGetLastError();
}

cudaError_t rb_lanes_fifo_scatter_prog(const float* d_staging, const rb_fifo_prog_job* d_jobs, uint32_t n_jobs, const rb_prog_op* d_ops,
                                       float* d_fifo, uint64_t stride, uint32_t* d_flags, cudaStream_t st) {
    if (n_jobs == 0) return cudaSuccess;
    k_fifo_scatter<true><<<n_jobs, 128, 0, st>>>(d_staging, d_jobs, d_fifo, stride, d_flags, d_ops);
    return cudaGetLastError();
}

cudaError_t rb_lanes_fifo_generate(const rb_fifo_gen_job* d_jobs, uint32_t n_jobs, const rb_prog_op* d_ops, const float* d_phase_in,
                                   float* d_phase_out, float* d_fifo, uint64_t stride, uint32_t* d_flags, cudaStream_t st) {
    if (n_jobs == 0) return cudaSuccess;
    k_fifo_generate<<<(n_jobs + GEN_PER_CTA - 1) / GEN_PER_CTA, GEN_THREADS, 0, st>>>(d_jobs, n_jobs, d_ops, d_phase_in, d_phase_out, d_fifo, stride, d_flags);
    return cudaGetLastError();
}

cudaError_t rb_lanes_fifo_compact(const float* d_src, float* d_dst, uint64_t stride, const uint32_t* d_drop, const uint32_t* d_keep,
                                  uint32_t n_streams, cudaStream_t st) {
    if (n_streams == 0) return cudaSuccess;
    k_fifo_compact<<<n_streams, 128, 0, st>>>(d_src, d_dst, stride, d_drop, d_keep);
    return cudaGetLastError();
}

cudaError_t rb_lanes_spread_flags(lanes::Row* d_rows, uint32_t n_rows, const uint32_t* d_row_stream, const lanes::Row* d_stream_rows, cudaStream_t st) {
    if (n_rows == 0) return cudaSuccess;
    k_spread_flags<<<(n_rows + 255) / 256, 256, 0, st>>>(d_rows, n_rows, d_row_stream, d_stream_rows);
    return cudaGetLastError();
}

cudaError_t rb_lanes_launch_classify(lanes::Row* d_rows, uint32_t n_rows, const uint8_t* d_row_channels, cudaStream_t st) {
    if (n_rows == 0) return cudaSuccess;
    k_classify_inputs<<<n_rows, 256, 0, st>>>(d_rows, n_rows, d_row_channels);
    return cudaGetLastError();
}
