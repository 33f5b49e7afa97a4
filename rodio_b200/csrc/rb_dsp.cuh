// rb_dsp.cuh — the arithmetic of rodio's per-sample adapters as device functions.
// Every float op is an explicitly rounded intrinsic (__fmul_rn/__fadd_rn/...), which nvcc never
// contracts into an FMA: rustc does not fuse a*b+c, and bit-parity with the reference depends on it.
// (The translation unit is additionally compiled with --fmad=false.)
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "rb_internal.h"

namespace rbd {

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float divf(float a, float b) { return __fdiv_rn(a, b); }

// src/math.rs:24-26 : first + (second - first) * numerator as f32 / denominator as f32
__device__ __forceinline__ float lerp(float first, float second, uint32_t numerator, uint32_t denominator) {
    float d = sub(second, first);
    float m = mul(d, __uint2float_rn(numerator));
    float q = divf(m, __uint2float_rn(denominator));
    return add(first, q);
}
// Same with the two u32->f32 casts hoisted by the caller.
__device__ __forceinline__ float lerp_f(float first, float second, float num_f, float den_f) {
    return add(first, divf(mul(sub(second, first), num_f), den_f));
}

// std::time::Duration::as_secs_f32 of `ns` nanoseconds: (secs as f32) + (nanos as f32) / 1e9
__device__ __forceinline__ float duration_secs_f32(uint64_t ns) {
    const uint64_t secs = ns / 1000000000ull;
    const uint32_t nanos = (uint32_t)(ns - secs * 1000000000ull);
    return add(__ull2float_rn(secs), divf(__uint2float_rn(nanos), 1000000000.0f));
}

// The closed-form per-sample adapters: k_distort / k_ramp / k_take (rb_kernels.cu) and the push programs of the sessions
// (k_fifo_scatter, rb_lanes.cu) run these bodies.  rb_session_host.h restates them for the CPU build in the same order.
// Distortion -- src/source/distortion.rs:66-72 : (x * gain).clamp(-t, t)   (f32::clamp: NaN passes through)
__device__ __forceinline__ float distort_sample(float x, float g, float t) {
    float v = mul(x, g);
    if (v < -t) v = -t;
    if (v > t) v = t;
    return v;
}
// LinearGainRamp -- src/source/linear_ramp.rs:79-104: the factor of a sample whose frame has seen `elapsed` ns
// (elapsed = frame * floor(1e9 / rate): the elapsed time advances once per frame while the ramp is running).
// after: the factor once the ramp is over (end with clamp_end, else 1.0); total_f = duration_secs_f32(total).
__device__ __forceinline__ float ramp_factor(uint64_t elapsed, uint64_t total, float start, float end, float after, float total_f) {
    float factor = after;
    if (elapsed < total) {
        const float p = divf(duration_secs_f32(elapsed), total_f);
        factor = add(mul(start, sub(1.0f, p)), mul(end, p));
    }
    return factor;
}
// TakeDuration's fade-out filter -- src/source/take.rs:34-41 on input sample `o` (o < count):
// sample * (remaining.as_millis() as f32) / (total.as_millis() as f32)
__device__ __forceinline__ float take_fade(float v, uint64_t o, uint64_t total, uint64_t dps, float total_ms) {
    const uint64_t remaining_ms = (total - o * dps) / 1000000ull;
    return divf(mul(v, __ull2float_rn(remaining_ms)), total_ms);
}

// ---- signal generators (a source, src/source/signal_generator.rs): k_siggen (rb_kernels.cu) and the generator fill of the
// sessions (k_fifo_generate, rb_lanes.cu)
// glibc's sinf for arguments in [0, 2*pi] -- what `(TAU * phase).sin()` (signal_generator.rs:51-53) resolves to on linux-gnu:
// the argument widened to double, one multiply-subtract of range reduction into [-pi/4, pi/4] with the quadrant, a degree-7
// (sine) or degree-8 (cosine) polynomial in double, one rounding to float.  The coefficients are the published ones of glibc
// >= 2.28 (sysdeps/ieee754/flt-32/sincosf_data.c); the restatement was held against the libm of this image on every float of
// [0, 0x40c90fdb] (tools/microbench/sinf_exhaustive.cpp: 1 086 918 620 arguments, 0 mismatches, with and without contraction of
// the double multiply-adds -- so the ifunc variant libm picks on the host does not matter).  FP64 here is IEEE: bit for bit.
__device__ __forceinline__ float sinf_glibc_0_tau(float y) {
    const double x = (double)y;
    const uint32_t top = (__float_as_uint(y) >> 20) & 0x7ffu;
    double xr, x2, sgn = 1.0;
    int n = 0;
    if (top < 0x3f4u) {                      // |y| < pi/4 (abstop12 of 0x1.921FB6p-1f)
        if (top < 0x398u) return y;          // |y| < 2^-12
        xr = x, x2 = __dmul_rn(x, x);
    } else {
        const double r = __dmul_rn(x, 0x1.45F306DC9C883p+23);               // 2/pi * 2^24
        n = (__double2int_rz(r) + 0x800000) >> 24;
        xr = __dsub_rn(x, __dmul_rn((double)n, 0x1.921FB54442D18p0));       // pi/2
        sgn = (n & 3) == 1 || (n & 3) == 2 ? -1.0 : 1.0;                     // sign[n & 3] = {1, -1, -1, 1}
        x2 = __dmul_rn(xr, xr);
        xr = __dmul_rn(xr, sgn);
    }
    const bool neg = (n & 2) != 0;           // second table: the cosine coefficients negated
    if ((n & 1) == 0) {
        const double s1c = -0x1.555545995a603p-3, s2c = 0x1.1107605230bc4p-7, s3c = -0x1.994eb3774cf24p-13;
        const double x3 = __dmul_rn(xr, x2);
        const double s1 = __dadd_rn(s2c, __dmul_rn(x2, s3c));
        const double x7 = __dmul_rn(x3, x2);
        const double s = __dadd_rn(xr, __dmul_rn(x3, s1c));
        return __double2float_rn(__dadd_rn(s, __dmul_rn(x7, s1)));
    }
    const double k = neg ? -1.0 : 1.0;
    const double c0 = k, c1 = k * -0x1.ffffffd0c621cp-2, c2k = k * 0x1.55553e1068f19p-5, c3 = k * -0x1.6c087e89a359dp-10,
                 c4 = k * 0x1.99343027bf8c3p-16;
    const double x4 = __dmul_rn(x2, x2);
    const double c2 = __dadd_rn(c3, __dmul_rn(x2, c4));
    const double c1v = __dadd_rn(c0, __dmul_rn(x2, c1));
    const double x6 = __dmul_rn(x4, x2);
    const double c = __dadd_rn(c1v, __dmul_rn(x4, c2k));
    return __double2float_rn(__dadd_rn(c, __dmul_rn(x6, c2)));
}
// signal_generator.rs:133, phase in [0, 1), step > 0: phase = (phase + step).rem_euclid(1.0).  SMALL (step < 1): q < 2, so q % 1.0
// is q or q - 1, both exact; otherwise q >= 0 and q - floor(q) is fmodf(q, 1.0f) exactly.  The step is 1 / (rate / freq) in f32,
// as the host computes it (rb_api.cu: plan_stream, rb_session_create_ex).
template <bool SMALL>
__device__ __forceinline__ float signal_phase_next(float phase, float step) {
    const float q = add(phase, step);
    return SMALL ? (q >= 1.0f ? sub(q, 1.0f) : q) : sub(q, floorf(q));
}
__device__ __forceinline__ float signal_value(uint32_t fn, float phase) {   // signal_generator.rs:51-69
    switch (fn) {
        case RB_SIGNAL_SINE: return sinf_glibc_0_tau(mul(6.2831855f, phase));
        case RB_SIGNAL_TRIANGLE: return sub(mul(4.0f, fabsf(sub(phase, floorf(add(phase, 0.5f))))), 1.0f);
        case RB_SIGNAL_SQUARE: return phase < 0.5f ? 1.0f : -1.0f;           // phase % 1.0 == phase inside [0, 1)
        default: return mul(2.0f, sub(phase, floorf(add(phase, 0.5f))));
    }
}
// src/source/blt.rs:558-560 : b0*x + b1*x1 + b2*x2 - a1*y1 - a2*y2, strictly left to right
__device__ __forceinline__ float biquad(float b0, float b1, float b2, float a1, float a2, float x, float x1, float x2,
                                        float y1, float y2) {
    float r = mul(b0, x);
    r = add(r, mul(b1, x1));
    r = add(r, mul(b2, x2));
    r = sub(r, mul(a1, y1));
    r = sub(r, mul(a2, y2));
    return r;
}
// Feed-forward half (no dependence on y): ((b0*x + b1*x1) + b2*x2)
__device__ __forceinline__ float biquad_ff(float b0, float b1, float b2, float x, float x1, float x2) {
    return add(add(mul(b0, x), mul(b1, x1)), mul(b2, x2));
}
// Recurrent half: (t - a1*y1) - a2*y2
__device__ __forceinline__ float biquad_fb(float a1, float a2, float t, float y1, float y2) {
    return sub(sub(t, mul(a1, y1)), mul(a2, y2));
}
// The same value with the two subtractions written as fma(p, -1, t) = RN(t - p): p * -1 is exact, so each step
// still rounds exactly once, but all three dependent operations now run on the FMA pipe.  An FMUL feeding an FADD
// crosses pipes (5 instead of 4 cycles each way): 18 cycles per sample for the serial chain instead of 12.
__device__ __forceinline__ float biquad_fb_chain(float a1, float a2, float t, float y1, float y2, float neg1) {
    return __fmaf_rn(mul(a2, y2), neg1, __fmaf_rn(mul(a1, y1), neg1, t));
}

// src/conversions/channels.rs:57-85 as a pure map: which input channel feeds output channel j
// (-1 = literal 0.0).
__device__ __forceinline__ int chan_map(uint32_t j, uint32_t c_in) {
    if (j < c_in) return (int)j;
    if (j == 1 && c_in == 1) return 0;
    return -1;
}

// Closed form of UniformSourceIterator (src/source/uniform.rs:50-97) =
// ChannelCountConverter(SampleRateConverter(Take(input))) re-bootstrapped per span chunk
// (src/conversions/sample_rate.rs:131-201, src/conversions/channels.rs:57-85).
// For output sample `o`: where the value comes from.  Exact integer math (the planner rejects
// from*to >= 2^32, so the reference's u32 products never wrap either).
struct UniformTap {
    uint64_t i0;     // flat input index of the left sample
    uint32_t num;    // interpolation numerator (0..to-1)
    uint32_t kind;   // 0: literal 0.0 (zero-filled channel), 1: x[i0] raw, 2: lerp(x[i0], x[i0 + c_in], num, to)
};
__device__ __forceinline__ UniformTap uniform_tap(const rb_uniform_params& u, uint32_t c_in, uint32_t c_out, uint64_t o) {
    UniformTap t;
    t.i0 = 0, t.num = 0, t.kind = 0;
    uint64_t base = 0;
    const rb_uniform_seg* seg = &u.tail;
    if (u.chunk_samples) {
        uint64_t k = u.full.out_samples ? o / u.full.out_samples : u.n_full_chunks;
        if (k >= u.n_full_chunks) k = u.n_full_chunks;
        else seg = &u.full;
        o -= k * u.full.out_samples;
        base = k * u.chunk_samples;
    }
    uint64_t fo = o / c_out;
    uint32_t j = (uint32_t)(o - fo * c_out);
    int c = chan_map(j, c_in);
    if (c < 0) return t;
    uint64_t q = fo * c_in + (uint32_t)c;            // position in the converter's flat output
    if (u.from == u.to) {
        t.i0 = base + q, t.kind = 1;
        return t;
    }
    uint64_t n;
    uint32_t ch;
    uint64_t full = seg->full_out_frames * c_in;
    if (q < full) {
        n = q / c_in;
        ch = (uint32_t)(q - n * c_in);
    } else {
        uint64_t r = q - full;
        uint64_t k = r / seg->p;
        n = seg->full_out_frames + k;
        ch = (uint32_t)(r - k * seg->p);
    }
    uint64_t frames_ch = seg->L + (ch < seg->p ? 1u : 0u);
    uint64_t prod = n * (uint64_t)u.from;
    uint64_t i = prod / u.to;
    t.num = (uint32_t)(prod - i * u.to);
    t.i0 = base + i * c_in + ch;
    t.kind = (i + 1 < frames_ch) ? 2u : 1u;
    return t;
}
__device__ __forceinline__ float uniform_sample(const float* __restrict__ x, const rb_uniform_params& u, uint32_t c_in,
                                                uint32_t c_out, float den_f, uint64_t o) {
    UniformTap t = uniform_tap(u, c_in, c_out, o);
    if (t.kind == 0) return 0.0f;
    float a = x[t.i0];
    if (t.kind == 1) return a;
    return lerp_f(a, x[t.i0 + c_in], __uint2float_rn(t.num), den_f);
}

// src/source/limit.rs:854-873 gain computer (dB of reduction wanted for this sample)
__device__ __forceinline__ float limiter_db(float sample, float threshold, float knee_width, float inv_knee_8) {
    const float LOG10_2 = 0.301029995663981195213738894724493027f;
    const float MIN_POSITIVE = 1.17549435e-38f;
    float lin = add(fabsf(sample), MIN_POSITIVE);
    float db = mul(mul(log2f(lin), LOG10_2), 20.0f);     // src/math.rs:87-90
    float bias_db = sub(db, threshold);
    float knee_boundary_db = mul(bias_db, 2.0f);
    if (knee_boundary_db < -knee_width) return 0.0f;
    if (fabsf(knee_boundary_db) <= knee_width) {
        float x = add(knee_boundary_db, knee_width);
        return mul(mul(x, x), inv_knee_8);
    }
    return bias_db;
}
// src/math.rs:52-56 : 2^(dB * 0.05 * LOG2_10)
__device__ __forceinline__ float db_to_linear(float decibels) {
    const float LOG2_10 = 3.32192809488736234787031942948939018f;
    return exp2f(mul(mul(decibels, 0.05f), LOG2_10));
}

// Rust float->int `as` casts: truncate, saturate, NaN -> 0 (what dasp_sample's conversions rely on).
__device__ __forceinline__ int32_t f32_as_i32(float v) { return __float2int_rz(v); }   // cvt.rzi.s32.f32 saturates, NaN->0
__device__ __forceinline__ int16_t f32_as_i16(float v) {
    int32_t i = __float2int_rz(v);
    i = max(-32768, min(32767, i));
    return (int16_t)i;
}
__device__ __forceinline__ int8_t f32_as_i8(float v) {
    int32_t i = __float2int_rz(v);
    i = max(-128, min(127, i));
    return (int8_t)i;
}

// dasp_sample 0.11.0 conv: X -> f32 (call site src/conversions/sample.rs:42-44)
__device__ __forceinline__ float load_as_f32(const void* p, uint32_t fmt, uint64_t i) {
    switch (fmt) {
        case RB_FMT_F32: return ((const float*)p)[i];
        case RB_FMT_I16: return divf((float)((const int16_t*)p)[i], 32768.0f);
        case RB_FMT_U16: return divf((float)((int32_t)((const uint16_t*)p)[i] - 32768), 32768.0f);
        case RB_FMT_I8: return divf((float)((const int8_t*)p)[i], 128.0f);
        case RB_FMT_U8: return divf((float)((int32_t)((const uint8_t*)p)[i] - 128), 128.0f);
        case RB_FMT_I32: return divf(__int2float_rn(((const int32_t*)p)[i]), 2147483648.0f);
        default: return divf(__int2float_rn(((const int32_t*)p)[i]), 8388608.0f);  // RB_FMT_I24_IN_I32
    }
}
// f32 -> X
__device__ __forceinline__ void store_from_f32(void* p, uint32_t fmt, uint64_t i, float s) {
    switch (fmt) {
        case RB_FMT_F32: ((float*)p)[i] = s; break;
        case RB_FMT_I16: ((int16_t*)p)[i] = f32_as_i16(mul(s, 32768.0f)); break;
        case RB_FMT_U16: ((uint16_t*)p)[i] = (uint16_t)((int32_t)f32_as_i16(mul(s, 32768.0f)) + 32768); break;
        case RB_FMT_I8: ((int8_t*)p)[i] = f32_as_i8(mul(s, 128.0f)); break;
        case RB_FMT_U8: ((uint8_t*)p)[i] = (uint8_t)((int32_t)f32_as_i8(mul(s, 128.0f)) + 128); break;
        case RB_FMT_I32: ((int32_t*)p)[i] = f32_as_i32(mul(s, 2147483648.0f)); break;
        default: ((int32_t*)p)[i] = f32_as_i32(mul(s, 8388608.0f)); break;
    }
}

}  // namespace rbd
