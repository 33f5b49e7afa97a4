// rb_session_host.h — the two FIFO / sum kernels of the streaming sessions (rb_lanes.cu: k_fifo_scatter, k_sum_slots) as plain
// host code, for the CPU build of the library's host code.  rb_api.cu includes it only when compiled with RB_SIMT_EMULATE
// (tests/emu/: rb_api.cu as C++ over a mock CUDA runtime, the lane kernels on the SIMT emulator), so that the session host code
// keeps running there; the CUDA build launches the kernels instead.  Same jobs, same order of the additions, one sample at a
// time.  The translation unit is compiled with -ffp-contract=off, like the kernels.
#pragma once
#include <cmath>
#include <limits>
#include <utility>
#include <vector>

#include "rb_lanes.h"
#include "rb_lanes_plan.h"

// The RESTART twins of the lane kernel (rb_lanes.cu: launch_restart_cc) on the SIMT emulator.  The session lists what its kernels
// may read (its own device buffers) in g_restart_readable before the launch; the ring starts out as NaN, so a cursor seeded wrongly
// behind a cut shows.
namespace session_host {
inline std::vector<std::pair<const char*, const char*>> g_restart_readable;
template <int CI, int CO, bool HASB, bool PRE, bool FRONT, bool DOWN, bool GUARD>
void restart_group(const lanes::Args& a, uint32_t g, simt::WarpEmu* w, float* ring) {
    simt::run_warp(w, [&] { lanes::warp_main<CI, CO, HASB, false, 1, false, PRE, FRONT, DOWN, GUARD, true>(a, g, ring); });
}
template <int CI, int CO>
void restart_cc(const lanes::Args& a, uint32_t g, simt::WarpEmu* w, float* ring, bool has_biquad, bool front) {
    const bool down = lanes::ratio_runs_down(a.from, a.to);
    if (front) down ? restart_group<CI, CO, true, false, true, true, false>(a, g, w, ring) : restart_group<CI, CO, true, false, true, false, false>(a, g, w, ring);
    else if (down) has_biquad ? restart_group<CI, CO, true, false, false, true, false>(a, g, w, ring) : restart_group<CI, CO, false, false, false, true, false>(a, g, w, ring);
    else has_biquad ? restart_group<CI, CO, true, true, false, false, true>(a, g, w, ring) : restart_group<CI, CO, false, true, false, false, true>(a, g, w, ring);
}
}  // namespace session_host

cudaError_t rb_lanes_launch_restart(const lanes::Args& a, uint32_t ch_in, uint32_t ch_out, bool has_biquad, bool front, cudaStream_t) {
    if (a.mix_len == 0 || a.n_groups == 0) return cudaSuccess;
    if (!a.cuts || !a.cut_first || a.from == a.to || (front && !has_biquad)) return cudaErrorInvalidValue;
    if (!((ch_in == 1 || ch_in == 2) && (ch_in == ch_out || (ch_in == 1 && ch_out == 2)))) return cudaErrorInvalidValue;
    simt::WarpEmu warp;
    warp.readable = session_host::g_restart_readable;
    constexpr int MAX_RS = lanes::Geo<2, 4>::RS;   // the largest ring of any variant
    std::vector<float> ring_store(32 * MAX_RS + 4);
    float* ring = ring_store.data();
    while ((uintptr_t)ring & 15) ring++;
    for (uint32_t g = 0; g < a.n_groups; g++) {
        for (int i = 0; i < 32 * MAX_RS; i++) ring[i] = std::numeric_limits<float>::quiet_NaN();
        if (ch_in == 2) session_host::restart_cc<2, 2>(a, g, &warp, ring, has_biquad, front);
        else if (ch_out == 2) session_host::restart_cc<1, 2>(a, g, &warp, ring, has_biquad, front);
        else session_host::restart_cc<1, 1>(a, g, &warp, ring, has_biquad, front);
    }
    return cudaSuccess;
}

cudaError_t rb_lanes_fifo_scatter(const float* staging, const rb_fifo_job* jobs, uint32_t n_jobs, float* fifo, uint64_t stride,
                                  uint32_t* flags, cudaStream_t) {
    for (uint32_t k = 0; k < n_jobs; k++) {
        const rb_fifo_job& j = jobs[k];
        for (uint64_t f = 0; f < j.frames; f++)
            for (uint32_t c = 0; c < j.ci; c++) {
                const float v = staging[j.src + f * j.src_ch + j.ch0 + c];
                if (!lanes::sample_in_class(v)) flags[j.row] = 1u;
                fifo[(uint64_t)j.row * stride + ((uint64_t)j.fill + f) * j.ci + c] = v;
            }
    }
    return cudaSuccess;
}

// rb_dsp.cuh's adapter bodies and rb_lanes.cu's run_prog, one rounding per operation (no contraction in this unit)
namespace session_host {
inline float duration_secs_f32(uint64_t ns) {
    const uint64_t secs = ns / 1000000000ull;
    const uint32_t nanos = (uint32_t)(ns - secs * 1000000000ull);
    return (float)secs + (float)nanos / 1000000000.0f;
}
inline float run_prog(float v, uint64_t n, uint32_t C, const rb_prog_op* ops, uint32_t n_ops) {
    for (uint32_t k = 0; k < n_ops; k++) {
        const rb_prog_op& op = ops[k];
        if (op.kind == RB_N_AMPLIFY) {
            v = v * op.p.amp;
        } else if (op.kind == RB_N_DISTORT) {
            v = v * op.p.dist.gain;
            if (v < -op.p.dist.threshold) v = -op.p.dist.threshold;
            if (v > op.p.dist.threshold) v = op.p.dist.threshold;
        } else if (op.kind == RB_N_RAMP) {
            const rb_ramp_params& r = op.p.ramp;
            const uint64_t elapsed = (n / C) * r.dt_ns;
            float factor = r.clamp_end ? r.end : 1.0f;
            if (elapsed < r.total_ns) {
                const float p = duration_secs_f32(elapsed) / duration_secs_f32(r.total_ns);
                factor = r.start * (1.0f - p) + r.end * p;
            }
            v = v * factor;
        } else {
            const rb_take_params& t = op.p.take;
            if (n < t.count) {
                if (t.fadeout) v = v * (float)((t.total_ns - n * t.dps_ns) / 1000000ull) / t.total_ms_f;
            } else {
                v = 0.0f;
            }
        }
    }
    return v;
}
}  // namespace session_host

cudaError_t rb_lanes_fifo_scatter_prog(const float* staging, const rb_fifo_prog_job* jobs, uint32_t n_jobs, const rb_prog_op* ops, float* fifo,
                                       uint64_t stride, uint32_t* flags, cudaStream_t) {
    for (uint32_t k = 0; k < n_jobs; k++) {
        const rb_fifo_job& j = jobs[k].j;
        for (uint64_t f = 0; f < j.frames; f++)
            for (uint32_t c = 0; c < j.ci; c++) {
                const uint64_t n = (jobs[k].base + f) * j.src_ch + j.ch0 + c;
                const float v = session_host::run_prog(staging[j.src + f * j.src_ch + j.ch0 + c], n, j.src_ch, ops + jobs[k].op0, jobs[k].n_ops);
                if (!lanes::sample_in_class(v)) flags[j.row] = 1u;
                fifo[(uint64_t)j.row * stride + ((uint64_t)j.fill + f) * j.ci + c] = v;
            }
    }
    return cudaSuccess;
}

// rb_dsp.cuh's generator (signal_phase_next, signal_value); the host's libm sinf is glibc's, which sinf_glibc_0_tau restates on
// [0, 2*pi] (tests/test_signal_generator.py::test_sinf_restatement_against_libm)
namespace session_host {
inline float signal_value(uint32_t fn, float phase) {
    switch (fn) {
        case RB_SIGNAL_SINE: return sinf(6.2831855f * phase);
        case RB_SIGNAL_TRIANGLE: return 4.0f * fabsf(phase - floorf(phase + 0.5f)) - 1.0f;
        case RB_SIGNAL_SQUARE: return phase < 0.5f ? 1.0f : -1.0f;
        default: return 2.0f * (phase - floorf(phase + 0.5f));
    }
}
}  // namespace session_host

cudaError_t rb_lanes_fifo_generate(const rb_fifo_gen_job* jobs, uint32_t n_jobs, const rb_prog_op* ops, const float* phase_in, float* phase_out,
                                   float* fifo, uint64_t stride, uint32_t* flags, cudaStream_t) {
    for (uint32_t k = 0; k < n_jobs; k++) {
        const rb_fifo_gen_job& j = jobs[k];
        float phase = phase_in[j.gen];
        for (uint32_t f = 0; f < j.frames; f++) {
            const float v = session_host::run_prog(session_host::signal_value(j.fn, phase), j.base + f, 1, ops + j.op0, j.n_ops);
            if (!lanes::sample_in_class(v)) flags[j.row] = 1u;
            fifo[(uint64_t)j.row * stride + j.fill + f] = v;
            const float q = phase + j.step;
            phase = j.step < 1.0f ? (q >= 1.0f ? q - 1.0f : q) : q - floorf(q);
        }
        phase_out[j.gen] = phase;
    }
    return cudaSuccess;
}

cudaError_t rb_lanes_launch_sum_slots(const float* partial, const uint32_t* slot, uint32_t n_groups, uint64_t pstride, uint64_t n_frames,
                                      uint32_t channels, float* out, cudaStream_t) {
    for (uint64_t f = 0; f < n_frames; f++)
        for (uint32_t j = 0; j < channels; j++) {
            float acc = 0.0f;
            for (uint32_t g = 0; g < n_groups; g++) {
                const uint32_t o = slot[g] & 0xffffu, w = slot[g] >> 16;
                if (j >= o && j < o + w) acc = acc + partial[(uint64_t)g * pstride + f * w + (j - o)];
            }
            out[f * channels + j] = acc;
        }
    return cudaSuccess;
}
