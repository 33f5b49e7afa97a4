// rb_master.cu — adapters on the MixerSource itself: Amplify(Limit(Amplify(mix))) (src/source/amplify.rs:63-65,
// src/source/limit.rs:854-988 around src/mixer.rs:70-136), in place on a rendered mix.
//
// One CTA walks the active runs of the mix as one sequence, in tiles of whole frames staged through shared memory:
//   - warp 0 (recurrence lanes): lane c runs channel c's integ / peak recurrence (limit.rs:909-913) over the frames of
//     tile t and overwrites the tile's limiter_db values with the peak after every update;
//   - warps 1.. (feed-forward workers): load tile t+1 with 16-byte loads, apply `pre`, compute limiter_db (limit.rs:854-873);
//     and for tile t-1 form the channel-coupled peak m at every sample from the stored trajectories, db_to_linear(-m),
//     `post`, store.
// The arithmetic is k_limit_tile's (rb_kernels.cu): the same rb_dsp.cuh functions and explicitly rounded intrinsics.
#include "rb_dsp.cuh"
#include "rb_internal.h"

using namespace rbd;

namespace {
constexpr int MT = 256;       // warp 0: recurrence lanes; warps 1..7: feed-forward workers
constexpr int NW = MT - 32;
constexpr int TS = 1920;      // samples per tile buffer: whole frames of 1..6, 8, 10 and 12 channels (TS / C frames otherwise)

// channel-coupled peak at sample (f, c): channels <= c after frame f's update, channels > c after frame f-1's
// (limit.rs:927-988: Mono -> peak, Stereo -> max(p0, p1), Multi -> fold(0.0, max))
__device__ __forceinline__ float coupled_peak(const float* cur, const float* prev, uint32_t c, uint32_t C) {
    if (C == 1) return cur[0];
    if (C == 2) return fmaxf(cur[0], c >= 1 ? cur[1] : prev[1]);
    float m = 0.0f;
    for (uint32_t j = 0; j < C; j++) m = fmaxf(m, j <= c ? cur[j] : prev[j]);
    return m;
}
}  // namespace

__global__ void __launch_bounds__(MT, 1) k_master(float* __restrict__ mix, const rb_master_run* __restrict__ runs, uint32_t n_runs,
                                                  uint64_t n_seq, uint32_t C, rb_master_params p, const float* __restrict__ state_in,
                                                  float* __restrict__ state_out) {
    __shared__ __align__(16) float s_x[3][TS];   // x * pre
    __shared__ __align__(16) float s_d[3][TS];   // limiter_db, overwritten by the peak after the frame's update
    __shared__ float s_carry[3][RB_MAX_CHANNELS];   // peaks after the last frame of a tile
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t TSC = (TS / C) * C;
    const uint64_t n_tiles = (n_seq + TSC - 1) / TSC;
    float integ = 0.0f, peak = 0.0f;
    if (warp == 0 && lane < C) {
        if (state_in) integ = state_in[lane], peak = state_in[C + lane];
        s_carry[2][lane] = peak;   // "tile -1"
    }
    const float rel = p.lim.release, att = p.lim.attack, omr = sub(1.0f, rel), oma = sub(1.0f, att);
    uint32_t r_ld = 0, r_st = 0;   // per-worker run cursors: a worker's sequence positions only grow
    auto mix_index = [&](uint32_t& r, uint64_t q) {
        while (r + 1 < n_runs && q >= runs[r].seq_end) r++;
        return q + runs[r].delta;
    };
    __syncthreads();
    for (uint64_t k = 0; k < n_tiles + 2; k++) {
        if (warp == 0) {
            const uint64_t t = k - 1;
            if (p.has_lim && k >= 1 && t < n_tiles && lane < C) {
                const uint32_t nf = (uint32_t)(min((uint64_t)TSC, n_seq - t * TSC) / C);
                float* d = s_d[t % 3] + lane;
                uint32_t f = 0;
                for (; f + 8 <= nf; f += 8) {
                    float l[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) l[u] = d[(f + u) * C];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const float in_c = fmaxf(l[u], add(mul(rel, integ), mul(omr, l[u])));   // limit.rs:909-912
                        integ = in_c;
                        peak = add(mul(att, peak), mul(oma, in_c));                            // limit.rs:913
                        l[u] = peak;
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) d[(f + u) * C] = l[u];
                }
                for (; f < nf; f++) {
                    const float l = d[f * C];
                    const float in_c = fmaxf(l, add(mul(rel, integ), mul(omr, l)));
                    integ = in_c;
                    peak = add(mul(att, peak), mul(oma, in_c));
                    d[f * C] = peak;
                }
                s_carry[t % 3][lane] = peak;
            }
        } else {
            const uint32_t w = tid - 32;
            if (k < n_tiles) {   // feed-forward of tile k
                const uint64_t base = k * TSC;
                const uint32_t cnt = (uint32_t)min((uint64_t)TSC, n_seq - base);
                float* xs = s_x[k % 3];
                float* ds = s_d[k % 3];
                for (uint32_t i = 4 * w; i < cnt; i += 4 * NW) {
                    const uint64_t q = base + i;
                    const uint64_t m0 = mix_index(r_ld, q);
                    float v[4];
                    if (i + 4 <= cnt && q + 4 <= runs[r_ld].seq_end && (m0 & 3u) == 0) {
                        const float4 x4 = __ldcg(reinterpret_cast<const float4*>(mix + m0));
                        v[0] = x4.x, v[1] = x4.y, v[2] = x4.z, v[3] = x4.w;
                    } else {
                        for (uint32_t u = 0; u < 4; u++) v[u] = (i + u < cnt) ? mix[mix_index(r_ld, q + u)] : 0.0f;
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        if (p.has_pre) v[u] = mul(v[u], p.pre);
                        xs[i + u] = v[u];
                        if (p.has_lim) ds[i + u] = limiter_db(v[u], p.lim.threshold, p.lim.knee, p.lim.inv_knee_8);
                    }
                }
            }
            if (k >= 2 && k - 2 < n_tiles) {   // gain and store of tile k-2
                const uint64_t t = k - 2;
                const uint64_t base = t * TSC;
                const uint32_t cnt = (uint32_t)min((uint64_t)TSC, n_seq - base);
                const float* xs = s_x[t % 3];
                const float* pk = s_d[t % 3];
                const float* carry = s_carry[(t + 2) % 3];
                for (uint32_t i = 4 * w; i < cnt; i += 4 * NW) {
                    float y[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        y[u] = xs[i + u];
                        if (i + u < cnt && p.has_lim) {
                            const uint32_t f = (i + u) / C, c = (i + u) - f * C;
                            const float* cur = pk + f * C;
                            const float m = coupled_peak(cur, f ? cur - C : carry, c, C);
                            y[u] = mul(y[u], db_to_linear(-m));
                        }
                        if (p.has_post) y[u] = mul(y[u], p.post);
                    }
                    const uint64_t q = base + i;
                    const uint64_t m0 = mix_index(r_st, q);
                    if (i + 4 <= cnt && q + 4 <= runs[r_st].seq_end && (m0 & 3u) == 0) {
                        *reinterpret_cast<float4*>(mix + m0) = make_float4(y[0], y[1], y[2], y[3]);
                    } else {
                        for (uint32_t u = 0; u < 4; u++)
                            if (i + u < cnt) mix[mix_index(r_st, q + u)] = y[u];
                    }
                }
            }
        }
        __syncthreads();
    }
    if (state_out && warp == 0 && lane < C) state_out[lane] = integ, state_out[C + lane] = peak;
}

cudaError_t rb_launch_master(float* mix, const rb_master_run* d_runs, uint32_t n_runs, uint64_t n_seq, uint32_t channels,
                             const rb_master_params& p, const float* state_in, float* state_out, cudaStream_t st) {
    if (channels == 0 || channels > RB_MAX_CHANNELS || n_seq % channels) return cudaErrorInvalidValue;
    if (n_seq == 0 && !state_out) return cudaSuccess;
    k_master<<<1, MT, 0, st>>>(mix, d_runs, n_runs, n_seq, channels, p, state_in, state_out);
    return cudaGetLastError();
}
