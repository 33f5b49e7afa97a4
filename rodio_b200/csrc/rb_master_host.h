// rb_master_host.h — the master chain (rb_master.cu) as plain host code, for the CPU build of the library's host code.
// rb_api.cu includes it only when compiled with RB_SIMT_EMULATE (tests/emu/: rb_api.cu as C++ over a mock CUDA runtime, the lane
// kernels on the SIMT emulator), so that the session host code keeps running there with a master chain; the CUDA build launches
// k_master instead.  Same recurrence, channel coupling and run table as the kernel, one sample at a time; the host's log2f /
// exp2f stand in for the device's (the emulator's session tests compare with the oracle by tolerance, splits with each other
// bit for bit).  The translation unit is compiled with -ffp-contract=off: no FMA, like the kernel.
#pragma once
#include <cmath>

#include "rb_internal.h"

cudaError_t rb_launch_master(float* mix, const rb_master_run* runs, uint32_t n_runs, uint64_t n_seq, uint32_t C, const rb_master_params& p,
                             const float* state_in, float* state_out, cudaStream_t) {
    if (C == 0 || C > RB_MAX_CHANNELS || n_seq % C) return cudaErrorInvalidValue;
    float integ[RB_MAX_CHANNELS] = {0}, peak[RB_MAX_CHANNELS] = {0};
    if (state_in)
        for (uint32_t c = 0; c < C; c++) integ[c] = state_in[c], peak[c] = state_in[C + c];
    const float rel = p.lim.release, att = p.lim.attack, omr = 1.0f - rel, oma = 1.0f - att;
    uint32_t r = 0;
    for (uint64_t q = 0; q < n_seq; q++) {
        while (r + 1 < n_runs && q >= runs[r].seq_end) r++;
        float& v = mix[q + runs[r].delta];
        const uint32_t c = (uint32_t)(q % C);
        const float x = p.has_pre ? v * p.pre : v;
        float y = x;
        if (p.has_lim) {   // limit.rs:854-873 (rb_dsp.cuh limiter_db), :909-913, :927-988
            const float lin = std::fabs(x) + 1.17549435e-38f;
            const float db = (std::log2(lin) * 0.301029995663981195213738894724493027f) * 20.0f;
            const float bias = db - p.lim.threshold, kb = bias * 2.0f;
            float ldb = bias;
            if (kb < -p.lim.knee) ldb = 0.0f;
            else if (std::fabs(kb) <= p.lim.knee) {
                const float t = kb + p.lim.knee;
                ldb = (t * t) * p.lim.inv_knee_8;
            }
            integ[c] = std::fmax(ldb, rel * integ[c] + omr * ldb);
            peak[c] = att * peak[c] + oma * integ[c];
            float m = peak[0];
            if (C == 2) m = std::fmax(peak[0], peak[1]);
            else if (C > 2) {
                m = 0.0f;
                for (uint32_t j = 0; j < C; j++) m = std::fmax(m, peak[j]);
            }
            y = x * std::exp2((-m * 0.05f) * 3.32192809488736234787031942948939018f);
        }
        v = p.has_post ? y * p.post : y;
    }
    if (state_out)
        for (uint32_t c = 0; c < C; c++) state_out[c] = integ[c], state_out[C + c] = peak[c];
    return cudaSuccess;
}
