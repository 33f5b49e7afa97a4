// rb_kernels.cu — one kernel per rodio adapter (the general, un-fused path) plus the mixer sum.
// Layout: every stream is a contiguous, 128-byte aligned run of interleaved f32 samples in HBM
// ("planar by stream", interleaved inside a stream exactly like rodio, src/source/mod.rs:131-135).
// Grid convention for the time-parallel kernels: blockIdx.x = node (stream) index, blockIdx.y walks
// tiles of that stream; consecutive threads touch consecutive samples (coalesced).
// The recurrences (biquad / AGC / limiter) keep the reference's sequential f32 order: one thread per
// independent chain, lanes = chains.  The fused kernels in rb_fused.cu are the fast path; these stay as
// the general path for arbitrary chains and as the cross-check (RB_NO_FUSION).
#include "rb_dsp.cuh"

using namespace rbd;

namespace {

constexpr int TPB = 256;
constexpr int TILE = TPB * 4;

// ---------------------------------------------------------------- time-parallel nodes
template <class F>
__device__ __forceinline__ void for_each_out(const rb_node_dev& nd, F f) {
    for (uint64_t base = (uint64_t)blockIdx.y * TILE; base < nd.n_out; base += (uint64_t)gridDim.y * TILE) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint64_t o = base + (uint64_t)k * TPB + threadIdx.x;
            if (o < nd.n_out) f(o);
        }
    }
}

__global__ void __launch_bounds__(TPB) k_convert(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = load_as_f32(nd.src, nd.fmt, o); });
}

__global__ void __launch_bounds__(TPB) k_amplify(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const float f = nd.p.amp.factor;
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = mul(x[o], f); });
}

// reverb: Mix(x, Delay(Amplify(x))) — src/source/mix.rs:43-53, delay.rs:68-75, amplify.rs:63-65
__global__ void __launch_bounds__(TPB) k_echo(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint64_t D = nd.p.echo.delay, L = nd.n_in;
    const float a = nd.p.echo.amplitude;
    for_each_out(nd, [&](uint64_t o) {
        float s2 = (o < D) ? 0.0f : mul(x[o - D], a);   // Delay emits literal 0.0 first
        float y = (o < L) ? add(x[o], s2) : s2;          // (Some, Some) => s1 + s2 ; (None, Some) => s2
        nd.dst[o] = y;
    });
}

// Mix of two sources (src/source/mix.rs:43-53; crossfade.rs:10-23 is built from it): s1 + s2 while both run, then whichever is left.
// Both inputs already went through their UniformSourceIterator (planner).  Second input: aux0, p.mix2.n2 samples.
__global__ void __launch_bounds__(TPB) k_mix2(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x1 = (const float*)nd.src;
    const float* __restrict__ x2 = nd.aux0;
    const uint64_t n1 = nd.n_in, n2 = nd.p.mix2.n2;
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = (o < n1 && o < n2) ? add(x1[o], x2[o]) : (o < n1 ? x1[o] : x2[o]); });
}

// Pausable (src/source/pausable.rs:85-97): `n` zeros (whole frames) in front of input sample `at`, everything behind them shifted
__global__ void __launch_bounds__(TPB) k_pause(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint64_t at = nd.p.pause.at, n = nd.p.pause.n;
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = o < at ? x[o] : (o < at + n ? 0.0f : x[o - n]); });
}

__global__ void __launch_bounds__(TPB) k_delay(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint64_t D = nd.p.echo.delay;
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = (o < D) ? 0.0f : x[o - D]; });
}

// ---------------------------------------------------------------- signal generators (a source, src/source/signal_generator.rs)
// A CTA owns SIG_GENS generators (4: the waveform -- ~100 instructions per sine -- is what the seven worker warps have to keep up
// with; with 32 generators per CTA the first version spent 220 cycles per sample step on 32 SMs, with 8 still 29).  The phase is a serial f32 recurrence per generator (`phase = (phase + step).rem_euclid(1.0)`,
// signal_generator.rs:133: it drifts by design, so it cannot be computed from the sample index): warp 0, lane = generator, walks
// it a tile ahead into shared memory; the other seven warps evaluate the waveform of the previous tile and store it with
// consecutive threads on consecutive samples.  Latency-bound by the recurrence (3 dependent operations per sample) -- input
// generation, outside every timed region.
constexpr int SIG_TILE = 256, SIG_THREADS = 256, SIG_PITCH = SIG_TILE + 1, SIG_GENS = 4;
__global__ void __launch_bounds__(SIG_THREADS) k_siggen(const rb_node_dev* __restrict__ nodes, uint32_t n_nodes) {
    __shared__ float s_phase[2][SIG_GENS * SIG_PITCH];
    const uint32_t g0 = blockIdx.x * SIG_GENS, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n_g = min((uint32_t)SIG_GENS, n_nodes - g0);
    uint64_t max_n = 0;
    for (uint32_t g = 0; g < n_g; g++) max_n = max(max_n, nodes[g0 + g].n_out);
    const uint64_t n_tiles = (max_n + SIG_TILE - 1) / SIG_TILE;
    float phase = 0.0f, step = 0.0f;
    if (warp == 0 && lane < n_g) step = nodes[g0 + lane].p.sig.step;
    for (uint64_t it = 0; it <= n_tiles; it++) {
        if (warp == 0) {
            if (it < n_tiles && lane < n_g) {
                float* row = &s_phase[it & 1][lane * SIG_PITCH];
                if (step < 1.0f) {
#pragma unroll 8
                    for (int t = 0; t < SIG_TILE; t++) {
                        row[t] = phase;
                        phase = signal_phase_next<true>(phase, step);
                    }
                } else {
                    for (int t = 0; t < SIG_TILE; t++) {
                        row[t] = phase;
                        phase = signal_phase_next<false>(phase, step);
                    }
                }
            }
        } else if (it > 0) {
            const uint64_t base = (it - 1) * SIG_TILE;
            // the tile's n_g * 128 values dealt out over the 224 worker threads: consecutive threads on consecutive samples
            for (uint32_t w = threadIdx.x - 32; w < n_g * SIG_TILE; w += SIG_THREADS - 32) {
                const uint32_t g = w / SIG_TILE, t = w % SIG_TILE;
                const rb_node_dev& nd = nodes[g0 + g];
                if (base + t < nd.n_out) nd.dst[base + t] = signal_value(nd.p.sig.fn, s_phase[(it - 1) & 1][g * SIG_PITCH + t]);
            }
        }
        __syncthreads();
    }
}

// Distortion — src/source/distortion.rs:66-72 : (x * gain).clamp(-t, t)   (f32::clamp: NaN passes through)
__global__ void __launch_bounds__(TPB) k_distort(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const float g = nd.p.dist.gain, t = nd.p.dist.threshold;
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = distort_sample(x[o], g, t); });
}

// LinearGainRamp / fade_in / fade_out — src/source/linear_ramp.rs:79-104.  Frame f sees
// elapsed = f * floor(1e9 / rate) ns (the elapsed time advances once per frame while the ramp is running).
__global__ void __launch_bounds__(TPB) k_ramp(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint64_t total = nd.p.ramp.total_ns, dt = nd.p.ramp.dt_ns;
    const float start = nd.p.ramp.start, end = nd.p.ramp.end;
    const float after = nd.p.ramp.clamp_end ? end : 1.0f;
    const float total_f = duration_secs_f32(total);
    const uint32_t C = nd.c_in;
    for_each_out(nd, [&](uint64_t o) {
        const float factor = ramp_factor((o / C) * dt, total, start, end, after, total_f);
        nd.dst[o] = mul(x[o], factor);
    });
}

// TakeDuration (+ fade-out filter) — src/source/take.rs:107-148,:34-41.  `count` input samples pass, then
// literal 0.0 pads the last frame.  Fade-out: sample * (remaining.as_millis() as f32) / (total.as_millis() as f32).
__global__ void __launch_bounds__(TPB) k_take(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint64_t total = nd.p.take.total_ns, dps = nd.p.take.dps_ns, count = nd.p.take.count;
    const float total_ms = nd.p.take.total_ms_f;
    const bool fade = nd.p.take.fadeout != 0;
    for_each_out(nd, [&](uint64_t o) {
        float v = 0.0f;                                   // Sample::EQUILIBRIUM padding
        if (o < count) {
            v = x[o];
            if (fade) v = take_fade(v, o, total, dps, total_ms);
        }
        nd.dst[o] = v;
    });
}

// ChannelVolume / Spatial — src/source/channel_volume.rs:71-88
__global__ void __launch_bounds__(TPB) k_chanvol(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint32_t ci = nd.c_in, co = nd.c_out;
    const float cif = (float)ci;
    for_each_out(nd, [&](uint64_t o) {
        uint64_t f = o / co;
        uint32_t j = (uint32_t)(o - f * co);
        const float* fr = x + f * ci;
        float m = 0.0f;                                  // Sample::EQUILIBRIUM
        for (uint32_t c = 0; c < ci; c++) m = add(m, fr[c]);
        m = divf(m, cif);
        nd.dst[o] = mul(m, nd.p.cv.vol[j]);
    });
}

// UniformSourceIterator = ChannelCountConverter(SampleRateConverter(Take(input))) — closed form
__global__ void __launch_bounds__(TPB) k_uniform(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float* __restrict__ x = (const float*)nd.src;
    const uint32_t ci = nd.c_in, co = nd.c_out;
    const rb_uniform_params& u = nd.p.uni;
    const float den_f = __uint2float_rn(u.to);
    for_each_out(nd, [&](uint64_t o) { nd.dst[o] = uniform_sample(x, u, ci, co, den_f, o); });
}

// ---------------------------------------------------------------- sequential recurrences
// One thread per (stream, channel) chain.
__global__ void __launch_bounds__(128) k_biquad_seq(const rb_node_dev* __restrict__ nodes, uint32_t n_nodes,
                                                    uint32_t max_c) {
    uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t s = gid / max_c, c = gid % max_c;
    if (s >= n_nodes) return;
    const rb_node_dev& nd = nodes[s];
    if (c >= nd.c_in) return;
    const float* __restrict__ x = (const float*)nd.src;
    float* __restrict__ y = nd.dst;
    float b0 = nd.p.blt.b0, b1 = nd.p.blt.b1, b2 = nd.p.blt.b2, a1 = nd.p.blt.a1, a2 = nd.p.blt.a2;
    const uint32_t C = nd.c_in;
    float x1 = 0.f, x2 = 0.f, y1 = 0.f, y2 = 0.f;
    uint32_t sw = 0;
    const uint32_t n_sw = nd.p.blt.n_sw;
    for (uint64_t i = c; i < nd.n_in; i += C) {      // flat position % C selects the state (blt.rs:472-476)
        while (sw < n_sw && i >= nd.p.blt.sw_at[sw]) {   // a span with another sample rate began: new coefficients, same state
            b0 = nd.p.blt.sw_k[sw][0], b1 = nd.p.blt.sw_k[sw][1], b2 = nd.p.blt.sw_k[sw][2], a1 = nd.p.blt.sw_k[sw][3], a2 = nd.p.blt.sw_k[sw][4];
            sw++;
        }
        float xv = x[i];
        float r = biquad(b0, b1, b2, a1, a2, xv, x1, x2, y1, y2);
        y2 = y1, x2 = x1, y1 = r, x1 = xv;
        y[i] = r;
    }
}

// ---- sequential adapters with coalesced memory traffic -------------------------------------------------
// One warp owns 32 streams (lane = stream, the reference's strict f32 order per stream).  Time advances in
// tiles of RT samples: the warp loads tile k+1 of all its streams with coalesced 128-byte requests (one
// stream per request, consecutive lanes on consecutive samples) into registers while every lane walks its
// own stream's tile k out of a padded shared-memory transpose; results go back through the same transpose
// and leave with coalesced stores.
constexpr int RT = 32;            // samples per tile (one 128-byte line per stream)
constexpr int RTS = RT + 1;       // padded row: lane r reading column k hits bank (r*33 + k) % 32 -> conflict-free

// AGC: state shared across interleaved channels (src/source/agc.rs:524-557 applies it to the flat stream).
// The reference's per-sample step splits into three passes with identical arithmetic (agc.rs:433-504):
//   A (sequential, cheap)  peak follower + running sum of squares           -> aux0 = sum[n], aux1 = peak[n]
//   B (time-parallel)      rms = sqrt(sum/8192); rms_gain; peak_gain; desired[n]     -> aux0 = desired[n]
//   C (sequential, cheap)  gain smoother + clamp, y = x * gain
// so the sqrt and the three IEEE divisions (≈ 500 cycles of dependent latency per sample in one thread)
// leave the sequential chains.
// Passes A and C as a warp-specialised pipeline (the shape of the fused mixer kernel): a CTA owns 32 streams,
// the mover warps stream tiles of AT samples per stream between HBM and shared memory with 16-byte accesses
// (stage L on tile k+1, stage S on tile k-1) while the chain warps (lane = stream) walk tile k.
// A single warp issues about one instruction every 3.5 cycles when every instruction hangs on a dependent chain,
// so the chain warps execute nothing but the recurrences: pass A runs its two independent chains on two warps
// (different SM sub-partitions), the movers apply y = x * gain on the way out of pass C.
//   A  sum[n]  = (sum - x[n-8192]^2) + x[n]^2                       (agc.rs:157; ring of 8192 squares)
//      peak[n] = |x| > peak ? |x| : peak * release + |x| * (1 - release)
//         (agc.rs:397-408 with coeff = 0 spelled out: peak * 0 = +0 and |x| * (1 - 0) = |x| exactly, peak >= +0)
//   C  k = desired > gain ? attack : release;  gain = clamp(gain * k + desired * (1 - k), 0.1, max_gain)
//         (agc.rs:474-491; desired is never NaN -- pass B builds it with fmin / fmax -- so min/max is the clamp)
constexpr int AT = 128;              // samples per stream and tile
constexpr int ATS = AT + 4;          // padded row, (AT + 4) / 4 odd: 16-byte accesses of 8 lanes hit 8 bank groups
constexpr int ANB = 3;               // tile ring: loading k+1, chains on k, storing k-1
constexpr int AGC_THREADS = 7 * 32;  // warps 3 (sub-partition 3) and, in pass A, 6 (sub-partition 2) are chain warps
constexpr size_t AGC_ARR = (size_t)32 * ATS;          // one array of a tile: [32 streams][ATS]
constexpr size_t AGC_BUF = 3 * AGC_ARR;               // x | x[n-8192] -> sum, or desired -> gain | peak
constexpr size_t AGC_SMEM = (size_t)ANB * AGC_BUF * sizeof(float);

template <int PASS>   // 0 = A, 2 = C
__global__ void __launch_bounds__(AGC_THREADS) k_agc_pipe(const rb_node_dev* __restrict__ nodes, uint32_t n_nodes) {
    extern __shared__ __align__(16) float agc_sm[];   // [ANB][3][32][ATS]
    __shared__ const float* s_in0[32];
    __shared__ const float* s_in1[32];
    __shared__ float* s_out0[32];
    __shared__ float* s_out1[32];
    __shared__ uint64_t s_n[32];
    __shared__ uint8_t s_al[32];     // every pointer of the row 16-byte aligned (a run of a from_iter source starts anywhere)
    __shared__ uint64_t s_max_n;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s0 = blockIdx.x * 32;
    const uint32_t cnt_rows = min(32u, n_nodes - s0);
    const rb_node_dev* nds = nodes + s0;
    if (threadIdx.x < 32) {
        uint64_t n = 0;
        if (lane < cnt_rows) {
            const rb_node_dev& nd = nds[lane];
            n = nd.n_in;
            s_in0[lane] = (const float*)nd.src;
            s_in1[lane] = PASS == 0 ? (const float*)nd.src - 8192 : nd.aux0;   // A: x[n-8192] (tiles below 8192 skip it), C: desired[n]
            s_out0[lane] = PASS == 0 ? nd.aux0 : nd.dst;
            s_out1[lane] = nd.aux1;
            s_al[lane] = (((uintptr_t)nd.src | (uintptr_t)nd.dst | (uintptr_t)nd.aux0 | (uintptr_t)nd.aux1) & 15u) == 0;
        } else {
            s_al[lane] = 1;
        }
        s_n[lane] = n;
        for (int o = 16; o; o >>= 1) n = max(n, __shfl_xor_sync(0xffffffffu, n, o));
        if (lane == 0) s_max_n = n;
    }
    __syncthreads();
    const uint64_t max_n = s_max_n;
    const uint32_t n_tiles = (uint32_t)((max_n + AT - 1) / AT);
    const bool chain_sum = warp == 3;                       // pass C: the gain chain
    const bool chain_peak = PASS == 0 && warp == 6;
    constexpr uint32_t NMOV = PASS == 0 ? 5 : 6;
    const uint32_t mv = warp < 3 ? warp : warp - 1;         // mover index among warps {0,1,2,4,5(,6)}

    // chain state (lane = stream)
    float gain = 1.0f, peak = 0.0f, sum = 0.0f;
    float attack = 0.f, release = 0.f, max_gain = 0.f, oma = 0.f, omr = 0.f;
    uint64_t my_n = 0;
    if ((chain_sum || chain_peak) && lane < cnt_rows) {
        const rb_node_dev& nd = nds[lane];
        my_n = nd.n_in;
        max_gain = nd.p.agc.max_gain, attack = nd.p.agc.attack, release = nd.p.agc.release;
        oma = sub(1.0f, attack), omr = sub(1.0f, release);
    }

    uint32_t lb = 0, cb = 0, sb = 0;   // ring slots of the tile being loaded / walked / stored
    for (uint32_t it = 0; it < n_tiles + 2; it++) {
        if (!chain_sum && !chain_peak) {
            if (it < n_tiles) {
                // ---- stage L: tile `it`, rows mv, mv+NMOV, ..: one 16-byte load per lane covers a row of AT samples ----
                const uint64_t n = (uint64_t)it * AT + 4 * lane;
                const bool second_on = PASS != 0 || (uint64_t)it * AT >= 8192;
                float* base = agc_sm + lb * AGC_BUF;
                // all of this warp's loads go out before the first one is consumed (HBM latency is paid once per tile)
                constexpr int NR = (32 + NMOV - 1) / NMOV;
                float4 vx[NR], vo[NR];
#pragma unroll
                for (int j = 0; j < NR; j++) {
                    const uint32_t r = mv + NMOV * j;
                    vx[j] = make_float4(0.f, 0.f, 0.f, 0.f), vo[j] = vx[j];
                    if (r >= 32) continue;
                    const uint64_t nr = s_n[r];
                    if (n + 4 <= nr && s_al[r]) {
                        vx[j] = __ldg(reinterpret_cast<const float4*>(s_in0[r] + n));
                        if (second_on) vo[j] = PASS == 0 ? __ldg(reinterpret_cast<const float4*>(s_in1[r] + n))
                                                         : *reinterpret_cast<const float4*>(s_in1[r] + n);
                    } else if (n < nr) {
                        float ax[4] = {0.f, 0.f, 0.f, 0.f}, ao[4] = {0.f, 0.f, 0.f, 0.f};
                        for (int k = 0; k < 4; k++)
                            if (n + k < nr) {
                                ax[k] = s_in0[r][n + k];
                                if (second_on) ao[k] = s_in1[r][n + k];
                            }
                        vx[j] = make_float4(ax[0], ax[1], ax[2], ax[3]), vo[j] = make_float4(ao[0], ao[1], ao[2], ao[3]);
                    }
                }
#pragma unroll
                for (int j = 0; j < NR; j++) {
                    const uint32_t r = mv + NMOV * j;
                    if (r >= 32) continue;
                    *reinterpret_cast<float4*>(base + r * ATS + 4 * lane) = vx[j];
                    *reinterpret_cast<float4*>(base + AGC_ARR + r * ATS + 4 * lane) = vo[j];
                }
            }
            if (it >= 2) {
                // ---- stage S: tile `it - 2` ----
                const uint64_t n = (uint64_t)(it - 2) * AT + 4 * lane;
                const float* base = agc_sm + sb * AGC_BUF;
                for (uint32_t r = mv; r < 32; r += NMOV) {
                    const uint64_t nr = s_n[r];
                    if (n >= nr) continue;
                    // pass A: sum (second array) -> aux0, peak (third array) -> aux1; pass C: x * gain -> dst
                    float4 a = *reinterpret_cast<const float4*>(base + (PASS == 0 ? AGC_ARR : 0) + r * ATS + 4 * lane);
                    const float4 b = *reinterpret_cast<const float4*>(base + (PASS == 0 ? 2 * AGC_ARR : AGC_ARR) + r * ATS + 4 * lane);
                    if (PASS == 2) a.x = mul(a.x, b.x), a.y = mul(a.y, b.y), a.z = mul(a.z, b.z), a.w = mul(a.w, b.w);
                    if (n + 4 <= nr && s_al[r]) {
                        *reinterpret_cast<float4*>(s_out0[r] + n) = a;
                        if (PASS == 0) *reinterpret_cast<float4*>(s_out1[r] + n) = b;
                    } else {
                        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
                        for (int j = 0; j < 4; j++)
                            if (n + j < nr) {
                                s_out0[r][n + j] = av[j];
                                if (PASS == 0) s_out1[r][n + j] = bv[j];
                            }
                    }
                }
            }
        } else if (it >= 1 && it <= n_tiles) {
            // ---- chains: tile `it - 1`, lane = stream; whole groups of four (positions past the end are never stored) ----
            const uint64_t n0 = (uint64_t)(it - 1) * AT;
            const int cnt = (int)min((uint64_t)AT, my_n > n0 ? my_n - n0 : 0);
            const float4* px = reinterpret_cast<const float4*>(agc_sm + cb * AGC_BUF + lane * ATS);
            float4* po = reinterpret_cast<float4*>(agc_sm + cb * AGC_BUF + AGC_ARR + lane * ATS);
            float4* pp = reinterpret_cast<float4*>(agc_sm + cb * AGC_BUF + 2 * AGC_ARR + lane * ATS);
            if (PASS == 0 && chain_sum) {
#pragma unroll 2
                for (int k4 = 0; k4 * 4 < cnt; k4++) {
                    const float4 a = px[k4], b = po[k4];
                    float4 o;
                    sum = add(sub(sum, mul(b.x, b.x)), mul(a.x, a.x)), o.x = sum;
                    sum = add(sub(sum, mul(b.y, b.y)), mul(a.y, a.y)), o.y = sum;
                    sum = add(sub(sum, mul(b.z, b.z)), mul(a.z, a.z)), o.z = sum;
                    sum = add(sub(sum, mul(b.w, b.w)), mul(a.w, a.w)), o.w = sum;
                    po[k4] = o;
                }
            } else if (PASS == 0) {
#pragma unroll 2
                for (int k4 = 0; k4 * 4 < cnt; k4++) {
                    const float4 a = px[k4];
                    const float av[4] = {a.x, a.y, a.z, a.w};
                    float r1[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const float v = fabsf(av[j]);
                        const float decayed = add(mul(peak, release), mul(v, omr));
                        peak = (v > peak) ? v : decayed;
                        r1[j] = peak;
                    }
                    pp[k4] = make_float4(r1[0], r1[1], r1[2], r1[3]);
                }
            } else {
#pragma unroll 2
                for (int k4 = 0; k4 * 4 < cnt; k4++) {
                    const float4 b = po[k4];
                    const float bv[4] = {b.x, b.y, b.z, b.w};
                    float r1[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const float desired = bv[j];
                        const bool up = desired > gain;
                        const float kk = up ? attack : release, omk = up ? oma : omr;
                        gain = add(mul(gain, kk), mul(desired, omk));
                        gain = fminf(fmaxf(gain, 0.1f), max_gain);
                        r1[j] = gain;
                    }
                    po[k4] = make_float4(r1[0], r1[1], r1[2], r1[3]);
                }
            }
        }
        if (it < n_tiles) lb = lb + 1 == ANB ? 0 : lb + 1;
        if (it >= 1 && it <= n_tiles) cb = cb + 1 == ANB ? 0 : cb + 1;
        if (it >= 2) sb = sb + 1 == ANB ? 0 : sb + 1;
        __syncthreads();
    }
}

// pass B: desired gain per sample, fully parallel (grid convention of the time-parallel kernels)
__global__ void __launch_bounds__(TPB) k_agc_desired(const rb_node_dev* __restrict__ nodes) {
    const rb_node_dev& nd = nodes[blockIdx.x];
    const float target = nd.p.agc.target, max_gain = nd.p.agc.max_gain, floor_v = nd.p.agc.floor;
    float* __restrict__ sums = nd.aux0;
    const float* __restrict__ peaks = nd.aux1;
    for_each_out(nd, [&](uint64_t o) {
        float rms = __fsqrt_rn(divf(sums[o], 8192.0f));                                  // agc.rs:413-418
        float rms_gain = (rms > 0.0f) ? divf(target, rms) : max_gain;
        float pk = peaks[o];
        float peak_gain = (pk > 0.0f) ? fminf(divf(target, pk), max_gain) : max_gain;    // agc.rs:424-431
        sums[o] = fmaxf(fminf(rms_gain, peak_gain), floor_v);
    });
}

// Limiter: per-channel envelope state, channel-coupled gain, sample-sequential (limit.rs:927-988).
// log2 (gain computer) and exp2 (dB -> linear) are feed-forward: evaluated LIM_K at a time around the
// short sequential envelope recurrences.
constexpr int LIM_K = 8;
__global__ void __launch_bounds__(32) k_limit_tile(const rb_node_dev* __restrict__ nodes, uint32_t n_nodes) {
    __shared__ float t_x[32 * RTS];
    const uint32_t lane = threadIdx.x;
    const uint32_t s0 = blockIdx.x * 32;
    const uint32_t cnt_rows = min(32u, n_nodes - s0);
    const rb_node_dev* nds = nodes + s0;
    uint64_t my_n = lane < cnt_rows ? nds[lane].n_in : 0;
    uint64_t max_n = my_n;
    for (int o = 16; o; o >>= 1) max_n = max(max_n, __shfl_xor_sync(0xffffffffu, max_n, o));
    float thr = 0.f, knee = 1.f, ik8 = 0.f, att = 0.f, rel = 0.f;
    uint32_t C = 1;
    if (lane < cnt_rows) {
        const rb_node_dev& nd = nds[lane];
        thr = nd.p.lim.threshold, knee = nd.p.lim.knee, ik8 = nd.p.lim.inv_knee_8;
        att = nd.p.lim.attack, rel = nd.p.lim.release, C = nd.c_in;
    }
    float integ[RB_MAX_CHANNELS], peaks[RB_MAX_CHANNELS];
    for (uint32_t c = 0; c < RB_MAX_CHANNELS; c++) integ[c] = 0.f, peaks[c] = 0.f;
    uint32_t c = 0;
    float rx[32];
    auto load_tile = [&](uint64_t n0) {
#pragma unroll
        for (int r = 0; r < 32; r++) {
            rx[r] = 0.0f;
            if ((uint32_t)r < cnt_rows) {
                const rb_node_dev& nd = nds[r];
                const uint64_t n = n0 + lane;
                if (n < nd.n_in) rx[r] = __ldg((const float*)nd.src + n);
            }
        }
    };
    load_tile(0);
    for (uint64_t n0 = 0; n0 < max_n; n0 += RT) {
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 32; r++) t_x[r * RTS + lane] = rx[r];
        __syncwarp();
        if (n0 + RT < max_n) load_tile(n0 + RT);
        const int cnt = (int)min((uint64_t)RT, my_n > n0 ? my_n - n0 : 0);
        float* mx = t_x + lane * RTS;
        for (int k0 = 0; k0 < cnt; k0 += LIM_K) {
            float xs[LIM_K], ldb[LIM_K], mp[LIM_K];
#pragma unroll
            for (int k = 0; k < LIM_K; k++) {
                xs[k] = mx[k0 + k];
                ldb[k] = limiter_db(xs[k], thr, knee, ik8);
            }
#pragma unroll
            for (int k = 0; k < LIM_K; k++) {
                mp[k] = 0.0f;
                if (k0 + k < cnt) {
                    float in_c = fmaxf(ldb[k], add(mul(rel, integ[c]), mul(sub(1.0f, rel), ldb[k])));   // limit.rs:909-912
                    integ[c] = in_c;
                    peaks[c] = add(mul(att, peaks[c]), mul(sub(1.0f, att), in_c));                       // limit.rs:913
                    float m;
                    if (C == 1) m = peaks[0];
                    else if (C == 2) m = fmaxf(peaks[0], peaks[1]);
                    else {
                        m = 0.0f;
                        for (uint32_t j = 0; j < C; j++) m = fmaxf(m, peaks[j]);
                    }
                    mp[k] = m;
                    c = (c + 1 == C) ? 0 : c + 1;
                }
            }
#pragma unroll
            for (int k = 0; k < LIM_K; k++)
                if (k0 + k < cnt) mx[k0 + k] = mul(xs[k], db_to_linear(-mp[k]));
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 32; r++) {
            if ((uint32_t)r < cnt_rows) {
                const rb_node_dev& nd = nds[r];
                const uint64_t n = n0 + lane;
                if (n < nd.n_in) nd.dst[n] = t_x[r * RTS + lane];
            }
        }
    }
}

// ---------------------------------------------------------------- mixer
// MixerSource::sum_current_sources (src/mixer.rs:185-198): acc = 0.0; for s in insertion order: acc += v_s.
// One thread per FOUR consecutive output samples (one 16-byte load per source when the source covers all
// four and is 16-byte aligned there, scalar loads otherwise); the loop over sources keeps the reference's
// order, loads are issued MIX_UNROLL sources at a time so enough bytes are in flight.  HBM-bound:
// algorithmic bytes = 4 * (sum of source samples + out_len).
constexpr int MIX_CHUNK = 256;   // sources staged per shared-memory chunk (pointer / start / len are block-uniform)
template <int U>
__global__ void __launch_bounds__(256) k_mix_ordered(const rb_mix_src* __restrict__ srcs, uint32_t n_srcs,
                                                     float* __restrict__ out, uint64_t out_len) {
    __shared__ rb_mix_src s_src[MIX_CHUNK];
    if (gridDim.y > 1) {   // run blockIdx.y of the source list -> its own partial row
        const uint32_t per = (n_srcs + gridDim.y - 1) / gridDim.y;
        const uint32_t first = min(n_srcs, blockIdx.y * per);
        srcs += first, n_srcs = min(per, n_srcs - first);
        out += (uint64_t)blockIdx.y * ((out_len + 3) & ~3ull);   // row pitch keeps the 16-byte stores aligned
    }
    const uint64_t n_quads = (out_len + 3) / 4;
    const uint64_t qd = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;   // grid covers every quad exactly once
    const bool live = qd < n_quads;
    const uint64_t p = qd * 4;
    float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f, acc3 = 0.0f;
    for (uint32_t base = 0; base < n_srcs; base += MIX_CHUNK) {
        const uint32_t cnt = min((uint32_t)MIX_CHUNK, n_srcs - base);
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) s_src[i] = srcs[base + i];
        __syncthreads();
        if (!live) continue;
        uint32_t s = 0;
        for (; s + U <= cnt; s += U) {
            float4 v[U];
            bool fast[U];
#pragma unroll
            for (int k = 0; k < U; k++) {
                const rb_mix_src& m = s_src[s + k];
                const uint64_t q = p - m.start;                       // wraps when p < start
                fast[k] = q < m.len && q + 3 < m.len && ((reinterpret_cast<uintptr_t>(m.data + q) & 15u) == 0);
                v[k] = fast[k] ? __ldg(reinterpret_cast<const float4*>(m.data + q)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int k = 0; k < U; k++) {
                if (fast[k]) {
                    acc0 = add(acc0, v[k].x), acc1 = add(acc1, v[k].y), acc2 = add(acc2, v[k].z), acc3 = add(acc3, v[k].w);
                } else {   // ragged edge / unaligned / a source that starts inside this quad
                    const rb_mix_src& m = s_src[s + k];
                    const uint64_t q = p - m.start;
                    if (q < m.len) acc0 = add(acc0, __ldg(m.data + q));
                    if (q + 1 < m.len) acc1 = add(acc1, __ldg(m.data + q + 1));
                    if (q + 2 < m.len) acc2 = add(acc2, __ldg(m.data + q + 2));
                    if (q + 3 < m.len) acc3 = add(acc3, __ldg(m.data + q + 3));
                }
            }
        }
        for (; s < cnt; s++) {
            const rb_mix_src& m = s_src[s];
            const uint64_t q = p - m.start;
            if (q < m.len) acc0 = add(acc0, __ldg(m.data + q));
            if (q + 1 < m.len) acc1 = add(acc1, __ldg(m.data + q + 1));
            if (q + 2 < m.len) acc2 = add(acc2, __ldg(m.data + q + 2));
            if (q + 3 < m.len) acc3 = add(acc3, __ldg(m.data + q + 3));
        }
    }
    if (!live) return;
    if (p + 3 < out_len) {
        *reinterpret_cast<float4*>(out + p) = make_float4(acc0, acc1, acc2, acc3);
    } else {
        if (p < out_len) out[p] = acc0;
        if (p + 1 < out_len) out[p + 1] = acc1;
        if (p + 2 < out_len) out[p + 2] = acc2;
    }
}

__global__ void __launch_bounds__(TPB) k_convert_flat(const void* __restrict__ in, uint32_t in_fmt, void* __restrict__ out,
                                                      uint32_t out_fmt, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        store_from_f32(out, out_fmt, i, load_as_f32(in, in_fmt, i));
}

}  // namespace

cudaError_t rb_launch_nodes(uint32_t kind, const rb_node_dev* d_nodes, uint32_t n_nodes, uint64_t max_n_out,
                            uint32_t max_channels, cudaStream_t st) {
    if (n_nodes == 0) return cudaSuccess;
    uint64_t tiles = (max_n_out + TILE - 1) / TILE;
    if (tiles < 1) tiles = 1;
    // enough blocks per stream to fill the machine, never more than the tiles there are
    uint64_t want = (132ull * 16 + n_nodes - 1) / n_nodes;
    if (want < 1) want = 1;
    uint32_t gy = (uint32_t)(tiles < want ? tiles : want);
    if (gy > 65535u) gy = 65535u;
    dim3 grid(n_nodes, gy);
    switch (kind) {
        case RB_N_CONVERT: k_convert<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_AMPLIFY: k_amplify<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_ECHO: k_echo<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_DELAY: k_delay<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_MIX2: k_mix2<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_PAUSE: k_pause<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_CHANVOL: k_chanvol<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_DISTORT: k_distort<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_RAMP: k_ramp<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_TAKE: k_take<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_UNIFORM: k_uniform<<<grid, TPB, 0, st>>>(d_nodes); break;
        case RB_N_BIQUAD: {
            if (max_channels < 1) max_channels = 1;
            uint32_t threads = n_nodes * max_channels;
            k_biquad_seq<<<(threads + 127) / 128, 128, 0, st>>>(d_nodes, n_nodes, max_channels);
            break;
        }
        case RB_N_AGC: {
            cudaError_t e = cudaFuncSetAttribute(k_agc_pipe<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AGC_SMEM);
            if (e == cudaSuccess) e = cudaFuncSetAttribute(k_agc_pipe<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AGC_SMEM);
            if (e != cudaSuccess) return e;
            k_agc_pipe<0><<<(n_nodes + 31) / 32, AGC_THREADS, AGC_SMEM, st>>>(d_nodes, n_nodes);
            k_agc_desired<<<grid, TPB, 0, st>>>(d_nodes);
            k_agc_pipe<2><<<(n_nodes + 31) / 32, AGC_THREADS, AGC_SMEM, st>>>(d_nodes, n_nodes);
            break;
        }
        case RB_N_LIMIT: k_limit_tile<<<(n_nodes + 31) / 32, 32, 0, st>>>(d_nodes, n_nodes); break;
        case RB_N_SIGNAL: k_siggen<<<(n_nodes + SIG_GENS - 1) / SIG_GENS, SIG_THREADS, 0, st>>>(d_nodes, n_nodes); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// ordered sum of the partial rows of the source runs
__global__ void __launch_bounds__(256) k_mix_sum_runs(const float* __restrict__ partial, uint32_t n_groups, uint64_t out_len,
                                                      float* __restrict__ out) {
    const uint64_t pitch = (out_len + 3) & ~3ull;
    for (uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; m < out_len; m += (uint64_t)gridDim.x * blockDim.x) {
        float acc = partial[m];
        for (uint32_t g = 1; g < n_groups; g++) acc = add(acc, partial[(uint64_t)g * pitch + m]);
        out[m] = acc;
    }
}

cudaError_t rb_launch_mix(const rb_mix_src* d_srcs, uint32_t n_srcs, float* d_out, uint64_t out_len, cudaStream_t st,
                          float* d_partial, uint32_t n_groups) {
    if (out_len == 0) return cudaSuccess;
    if (d_partial && n_groups > 1) {
        const uint64_t nq = (out_len + 3) / 4;
        const dim3 grid((uint32_t)((nq + 255) / 256), n_groups);
        k_mix_ordered<16><<<grid, 256, 0, st>>>(d_srcs, n_srcs, d_partial, out_len);
        const uint64_t sb = (out_len + 255) / 256;
        k_mix_sum_runs<<<(uint32_t)(sb < 1184 ? sb : 1184), 256, 0, st>>>(d_partial, n_groups, out_len, d_out);
        return cudaGetLastError();
    }
    // one thread per 4 outputs; the fewer threads there are, the more 16-byte loads each keeps in flight
    const uint64_t n_quads = (out_len + 3) / 4;
    const uint64_t blocks = (n_quads + 255) / 256;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
    if (n_quads >= 96 * 1024) k_mix_ordered<8><<<(uint32_t)blocks, 256, 0, st>>>(d_srcs, n_srcs, d_out, out_len);
    else k_mix_ordered<16><<<(uint32_t)blocks, 256, 0, st>>>(d_srcs, n_srcs, d_out, out_len);
    return cudaGetLastError();
}

cudaError_t rb_launch_convert(const void* d_in, uint32_t in_fmt, void* d_out, uint32_t out_fmt, uint64_t n,
                              cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    uint64_t blocks = (n + TPB - 1) / TPB;
    if (blocks > 132ull * 16) blocks = 132ull * 16;
    k_convert_flat<<<(uint32_t)blocks, TPB, 0, st>>>(d_in, in_fmt, d_out, out_fmt, n);
    return cudaGetLastError();
}
