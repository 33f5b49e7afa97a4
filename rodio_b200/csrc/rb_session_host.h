// rb_session_host.h — the two FIFO / sum kernels of the streaming sessions (rb_lanes.cu: k_fifo_scatter, k_sum_slots) as plain
// host code, for the CPU build of the library's host code.  rb_api.cu includes it only when compiled with RB_SIMT_EMULATE
// (tests/emu/: rb_api.cu as C++ over a mock CUDA runtime, the lane kernels on the SIMT emulator), so that the session host code
// keeps running there; the CUDA build launches the kernels instead.  Same jobs, same order of the additions, one sample at a
// time.  The translation unit is compiled with -ffp-contract=off, like the kernels.
#pragma once
#include "rb_lanes.h"
#include "rb_lanes_plan.h"

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
