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
