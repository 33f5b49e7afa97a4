// rb_internal.h — structures shared by the host planner (rb_api.cu) and the kernels (rb_kernels.cu).
// Product code: never includes anything under oracle/.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/rodio_b200.h"

#define RB_MAX_CHANNELS 12
#define RB_UNIFORM_SPAN_CAP 32768u
#define RB_MAX_BLT_SWITCH 3          // format changes inside one source that a filter follows (4 buffers)   // reference src/source/uniform.rs:56

// Internal node kinds (one per kernel family).
enum rb_node_kind : uint32_t {
    RB_N_CONVERT = 0,   // sample format -> f32        (src/conversions/sample.rs:42-44)
    RB_N_AMPLIFY = 1,   // x * factor                   (src/source/amplify.rs:63-65)
    RB_N_BIQUAD = 2,    // DF1 biquad                   (src/source/blt.rs:558-560)
    RB_N_ECHO = 3,      // x[n] + a*x[n-D]              (src/source/mod.rs:628-634)
    RB_N_DELAY = 4,     // D zeros then x               (src/source/delay.rs:68-75)
    RB_N_AGC = 5,       // src/source/agc.rs:433-504
    RB_N_LIMIT = 6,     // src/source/limit.rs:854-988
    RB_N_CHANVOL = 7,   // src/source/channel_volume.rs:71-88 (also Spatial)
    RB_N_UNIFORM = 8,   // src/source/uniform.rs + conversions/{sample_rate,channels}.rs
    RB_N_DISTORT = 9,   // src/source/distortion.rs:66-72
    RB_N_RAMP = 10,     // src/source/linear_ramp.rs:79-104 (also fade_in / fade_out)
    RB_N_TAKE = 11,     // src/source/take.rs:107-148 (+ fade-out filter :34-41)
    RB_N_SIGNAL = 12,   // src/source/signal_generator.rs:107-135 (a source: no input)
    RB_N_MIX2 = 13,     // src/source/mix.rs:43-53 (second input: aux0, p.mix2.n2 samples)
    RB_N_PAUSE = 14,    // src/source/pausable.rs:85-97: p.pause.n zeros in front of input sample p.pause.at
    RB_N_KINDS = 15
};

// Closed-form description of one UniformSourceIterator application.
// The input is cut into re-bootstrap chunks of `chunk_samples` (uniform.rs:56,:83-96); every chunk is an
// independent SampleRateConverter + ChannelCountConverter run.  A chunk (or the whole input) may end in an
// incomplete frame of p < channels samples (odd delay on stereo, odd mono span feeding a stereo adapter):
// the converter then keeps L+1 frames for channels < p and L for the rest (zip truncation,
// sample_rate.rs:174-178,:195-199), and ChannelCountConverter regroups the flat result (channels.rs:57-85).
struct rb_uniform_seg {
    uint64_t L;                   // whole input frames in the segment
    uint32_t p;                   // samples of the trailing incomplete frame
    uint32_t pad_;
    uint64_t full_out_frames;     // converter output frames in which every channel has a value
    uint64_t flat_total;          // samples the SampleRateConverter yields for the segment
    uint64_t out_samples;         // samples after ChannelCountConverter
};
struct rb_uniform_params {
    uint32_t from, to;            // gcd-reduced rates (sample_rate.rs:74); from == to -> pass-through
    uint64_t chunk_samples;       // 0 = the whole input is one segment (`tail`)
    uint64_t n_full_chunks;
    rb_uniform_seg full;          // every full chunk
    rb_uniform_seg tail;          // the last, shorter chunk (or the whole input)
};

// Limiter coefficients (src/source/limit.rs:94-130, :854-988); attack / release for the rate the limiter was built at.
struct rb_lim_params { float threshold, knee, inv_knee_8, attack, release; };

// The closed-form per-sample adapters (rb_dsp.cuh): the general kernels and the push programs of the sessions share them.
struct rb_dist_params { float gain, threshold; };
struct rb_ramp_params { uint64_t total_ns, dt_ns; float start, end; uint32_t clamp_end; };
struct rb_take_params { uint64_t total_ns, dps_ns, count; float total_ms_f; uint32_t fadeout; };

// One adapter applied to one stream, as the device sees it.  POD, 16-byte aligned.
struct alignas(16) rb_node_dev {
    const void* src;       // f32 except for RB_N_CONVERT
    float* dst;
    uint64_t n_in;         // samples
    uint64_t n_out;        // samples
    uint32_t c_in, c_out;  // channels
    uint32_t kind;
    uint32_t fmt;          // rb_sample_format of src (RB_N_CONVERT)
    float* aux0;           // per-stream scratch rows (same capacity as dst) for multi-pass adapters (AGC)
    float* aux1;
    union {
        struct { float factor; } amp;
        struct {
            float b0, b1, b2, a1, a2;
            uint32_t n_sw;                       // coefficient changes at span boundaries (blt.rs:122-137): from flat sample sw_at[k] on, sw_k[k]
            uint64_t sw_at[RB_MAX_BLT_SWITCH];
            float sw_k[RB_MAX_BLT_SWITCH][5];
        } blt;
        struct { uint64_t delay; float amplitude; } echo;
        struct { float target, max_gain, floor, attack, release; } agc;
        rb_lim_params lim;
        struct { float vol[RB_MAX_CHANNELS]; } cv;
        rb_dist_params dist;
        rb_ramp_params ramp;
        rb_take_params take;
        struct { float step; uint32_t fn; } sig;
        struct { uint64_t n2; } mix2;
        struct { uint64_t at, n; } pause;
        rb_uniform_params uni;
    } p;
};

// One mixer input as the mix kernel sees it.
struct rb_mix_src {
    const float* data;   // uniform (mixer rate / channels) samples of this stream
    uint64_t start;      // first mixer output sample it contributes to (frame aligned)
    uint64_t len;        // samples
};

// ---- launchers implemented in rb_kernels.cu (all asynchronous on `st`) ----
cudaError_t rb_launch_nodes(uint32_t kind, const rb_node_dev* d_nodes, uint32_t n_nodes, uint64_t max_n_out,
                            uint32_t max_channels, cudaStream_t st);
// n_groups > 1: the source list is cut into n_groups contiguous runs summed concurrently into d_partial
// ([n_groups][out_len]) and the runs are added in order -- more bytes in flight when there are few output samples.
cudaError_t rb_launch_mix(const rb_mix_src* d_srcs, uint32_t n_srcs, float* d_out, uint64_t out_len, cudaStream_t st,
                          float* d_partial = nullptr, uint32_t n_groups = 1);
cudaError_t rb_launch_convert(const void* d_in, uint32_t in_fmt, void* d_out, uint32_t out_fmt, uint64_t n,
                              cudaStream_t st);

// ---- adapters on the MixerSource itself: Amplify(Limit(Amplify(mix))), each stage optional (rb_master.cu) ----
struct rb_master_params {
    float pre, post;                     // 1.0 where the AMPLIFY is absent
    uint32_t has_pre, has_lim, has_post;
    rb_lim_params lim;                   // built for the mixer's rate
};
// The active runs of the mix (where MixerSource::next() returns Some) are one sequence for the chain; a gap is not pulled.
// Run r covers sequence samples [runs[r-1].seq_end, runs[r].seq_end) at mix samples seq + runs[r].delta.
struct rb_master_run {
    uint64_t seq_end;
    uint64_t delta;
};
// In place on `mix`.  n_seq = total samples of the runs (whole frames of `channels`).  state_in: integ[channels] then
// peak[channels] (nullptr: zero, a new limiter); state_out (may be nullptr) receives the state after the last frame.
cudaError_t rb_launch_master(float* mix, const rb_master_run* d_runs, uint32_t n_runs, uint64_t n_seq, uint32_t channels,
                             const rb_master_params& p, const float* state_in, float* state_out, cudaStream_t st);
