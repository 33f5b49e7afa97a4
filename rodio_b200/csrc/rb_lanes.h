// rb_lanes.h — interface between the fused planner (rb_fused.cu) and the lane-per-stream kernel (rb_lanes.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "rb_internal.h"
#include "rb_lanes_core.h"

// One stream of a batch that fits the lane kernel's shape (C = 1 or 2 interleaved channels, the mixer has the same C):
//   f32 source -> UniformSourceIterator(C ch, to) with reduced from < to -> [biquad] -> [one gain] -> mixer(C ch)
struct rb_lanes_stream {
    const float* in;       // device, 16-byte aligned, 16-byte tail pad
    uint64_t n_frames;
    uint64_t out_len;      // frames
    uint64_t mix_start;    // frames
    uint32_t from, to;     // reduced rate pair of this stream, from <= to (1:1 = already at the mixer's rate)
    uint32_t channels;     // of this stream: the mixer's, or 1 in a stereo mixer (the sample is repeated on both channels)
    float b0, b1, b2, a1, a2;
    float post;
    float pre;             // gain in front of the conversion (has_pre)
    float mid;             // front: gain between the filter and the conversion
};

struct rb_lanes_plan;

// *out stays NULL when the shape is not covered.  `d_out` is the mixer output ([mix_len] f32).
// mix_len in frames; `d_out` holds mix_len * channels floats.  Streams with different rate pairs are served class by
// class (rb_lanes_plan.h classes_by_ratio): the mixer sum then groups by class first.
// mode: LANES_TIME_PARALLEL asks for the time-parallel biquad plan (built only when the batch qualifies: rb_lanes_batch.cu),
// LANES_NO_DUO keeps every class on k_fused_lanes (A/B runs; the environment variable RB_NO_DUO does the same).
enum : uint32_t { LANES_TIME_PARALLEL = 1u, LANES_NO_DUO = 2u, LANES_ONE_GROUP = 4u, LANES_NO_LERPMIX = 8u };   // ONE_GROUP: k_lerp_mix sums all streams in one
                                                                                       // sequential chain (the reference's order, bit for bit)
cudaError_t rb_lanes_try_create(const rb_lanes_stream* streams, size_t n_streams, uint32_t channels, bool has_biquad, bool has_post,
                                bool has_pre, bool front, float* d_out, uint64_t mix_len, int sm_count, cudaStream_t st, rb_lanes_plan** out,
                                uint32_t mode = 0);
// 2: k_fused_lanes, 3: every class on k_fused_duo, 4: the time-parallel plan (k_fused_duo over segment rows),
// 6: k_lerp_mix (filter-free chains, parallel over the timeline)
int rb_lanes_kind(const rb_lanes_plan* p);
// streams per partial sum of the mixer: 32 (k_fused_lanes) or 64 (k_fused_duo: lane = even row + odd row, then the same tree)
uint32_t rb_lanes_mix_group(const rb_lanes_plan* p);
// time-parallel plan: number of timeline segments, their length and the warm-up in front of each (frames); zeros otherwise
void rb_lanes_tp_geometry(const rb_lanes_plan* p, uint32_t* segments, uint32_t* seg_len, uint32_t* warmup);
// Inputs were (re)written: classify them again before the next render.
void rb_lanes_inputs_changed(rb_lanes_plan* p);
cudaError_t rb_lanes_run(rb_lanes_plan* p, cudaStream_t st);
uint32_t rb_lanes_launch_count(const rb_lanes_plan* p);
void rb_lanes_destroy(rb_lanes_plan* p);

// ---- streaming blocks (rb_session_* in rb_api.cu): the caller owns every buffer and fills lanes::Args itself ----
// k_fused_lanes over a.rows (one class: one rate pair -- a.from == a.to selects the pass-through variant --, ch_in channels
// per stream, ch_out channels in the mixer) ...
cudaError_t rb_lanes_launch_kernel(const lanes::Args& a, uint32_t ch_in, uint32_t ch_out, bool has_biquad, bool ff2, bool has_post,
                                   bool has_pre, bool front, bool guard, cudaStream_t st);
// The same launch for a class some row of which changes its converter run inside the block, any number of times (a.cuts and
// a.cut_first, rb_lanes_core.h: Cut; never a same-rate class).  Rows, groups and the bits of rows without a cut are those of rb_lanes_launch_kernel.
cudaError_t rb_lanes_launch_restart(const lanes::Args& a, uint32_t ch_in, uint32_t ch_out, bool has_biquad, bool front, cudaStream_t st);
// k_fused_duo (rb_duo_core.h) over a.rows: mono sources below the mixer's rate, two rows per lane, a.n_groups groups of 64
cudaError_t rb_duo_launch_kernel(const lanes::Args& a, bool has_biquad, bool ff2, bool has_post, cudaStream_t st);
// ---- k_lerp_mix (rb_lanes.cu): resample -> [one gain] -> mixer sum for chains WITHOUT a filter, parallel over the timeline ----
// Nothing is carried from sample to sample in such a chain, so a thread owns timeline positions, walks the streams of its group
// in insertion order and adds them up in a register: no shared memory, no cross-lane traffic, and the sum inside a group IS the
// reference's sequential sum (src/mixer.rs:185-198).  All streams of the launch share one reduced rate pair and one phase
// (mix_start modulo `to`), so the input offset and the numerator of a timeline position are the same for every stream.
struct rb_lerpmix_row {      // one stream, 32 bytes
    const float* p;          // input, shifted so that p[idx] is the left tap of the timeline position whose table entry is idx
    uint32_t lo, hi_int, hi; // timeline frames [lo, hi_int) interpolate, [hi_int, hi) emit the last frame raw
    float post;              // the one gain (1.0: none)
    uint32_t row;            // index into the lanes::Row array (classification verdict: Row::flags)
    uint32_t pad_;
};
struct rb_lerpmix_args {
    const rb_lerpmix_row* rows;
    const lanes::Row* lane_rows;   // flags (ROW_UNSAFE) per stream
    uint32_t n_rows, rows_per_group, n_groups;
    uint32_t from, to;
    uint64_t origin;               // timeline frame whose numerator is 0 for every stream (the common phase)
    float den_f, rcp_den;
    uint64_t mix_len;
    float* out;                    // [n_groups][pstride] (n_groups == 1: the mixer output itself)
    uint64_t pstride;
    uint32_t has_post;
};
cudaError_t rb_lerpmix_launch(const rb_lerpmix_args& a, cudaStream_t st);
// ... and the ordered sum of n_groups partial rows (all classes) into d_out[0, n_floats).
cudaError_t rb_lanes_launch_sum(const float* d_partial, uint32_t n_groups, uint64_t pstride, uint64_t n_floats, float* d_out,
                                cudaStream_t st);
// ---- the FIFOs and the mixer sum of the streaming sessions: one FIFO, one filter state and one input flag per SLOT ROW ----
// A session source of CI channels feeds k = min(CI, mixer channels) of the mixer's channels; its rows carry channels
// (2s, 2s + 1) as CI = CO = 2 rows and an odd last channel as a CI = CO = 1 row (a mono source in a wider mixer: one CI = 1,
// CO = 2 row on channels 0 and 1).  A row's FIFO holds its `ci` channels interleaved.
struct rb_fifo_job {          // one row of one push, 24 bytes
    uint64_t src;             // float offset of the source's first new frame in the staging buffer
    uint32_t row;             // FIFO (fifo + row * stride) and flag of the row
    uint32_t frames, fill;    // new frames; frames already in the row's FIFO
    uint8_t src_ch, ch0, ci;  // the source's interleaving; the first source channel the row carries, and how many (1 or 2)
    uint8_t pad_;
};
// FIFO scatter: every job appends `frames` frames of channels [ch0, ch0 + ci) of its source behind the row's fill frames;
// flags[row] becomes non-zero (and stays so) when one of them lies outside the exact-reciprocal class.  One CTA per job.
cudaError_t rb_lanes_fifo_scatter(const float* d_staging, const rb_fifo_job* d_jobs, uint32_t n_jobs, float* d_fifo, uint64_t stride,
                                  uint32_t* d_flags, cudaStream_t st);
// ---- push programs: the closed-form adapters a source's chain begins with (rb_dsp.cuh), applied as the PCM is pushed ----
// kind: RB_N_AMPLIFY, RB_N_RAMP, RB_N_TAKE or RB_N_DISTORT (rb_internal.h), with the parameters the batch planner gives them.
struct rb_prog_op {
    uint32_t kind, pad_;
    union {
        float amp;
        rb_dist_params dist;
        rb_ramp_params ramp;
        rb_take_params take;
    } p;
};
struct rb_fifo_prog_job {     // a job of a session with push programs, 40 bytes
    rb_fifo_job j;
    uint64_t base;            // frames of the source that went through its program before this push
    uint32_t op0, n_ops;      // the source's program: ops[op0, op0 + n_ops) (n_ops = 0: none)
};
// The same scatter with every sample n = (base + f) * src_ch + ch0 + c of the source first run through the job's program, in
// chain order, and classified after it.
cudaError_t rb_lanes_fifo_scatter_prog(const float* d_staging, const rb_fifo_prog_job* d_jobs, uint32_t n_jobs, const rb_prog_op* d_ops,
                                       float* d_fifo, uint64_t stride, uint32_t* d_flags, cudaStream_t st);
// ---- generator sources (RB_FX_SIGNAL): the session writes their samples into the FIFO itself, before each render ----
struct rb_fifo_gen_job {      // one generator, 40 bytes
    uint64_t base;            // samples it has generated so far: the index of its next sample in the source and its program
    uint32_t row, fill;       // its row (mono: one per generator) and the frames already in that row's FIFO
    uint32_t frames;          // samples to generate now (0: the phase passes through unchanged)
    uint32_t gen;             // its phase slot
    uint32_t op0, n_ops;      // its push program: ops[op0, op0 + n_ops)
    uint32_t fn;              // rb_signal_function
    float step;               // 1 / (rate / frequency) in f32 (signal_generator.rs:118-119)
};
// Generator fill: job k writes samples [base, base + frames) of its generator behind the row's fill frames -- the phase recurrence
// from phase_in[gen], the waveform, the program, the sticky classification into flags[row] -- and leaves the phase of its next
// sample in phase_out[gen].  A few generators per CTA; every job, with or without frames, writes its phase_out.
cudaError_t rb_lanes_fifo_generate(const rb_fifo_gen_job* d_jobs, uint32_t n_jobs, const rb_prog_op* d_ops, const float* d_phase_in,
                                   float* d_phase_out, float* d_fifo, uint64_t stride, uint32_t* d_flags, cudaStream_t st);
// FIFO compaction into the other arena: dst[r][0, keep[r]) = src[r][drop[r], drop[r] + keep[r]).
cudaError_t rb_lanes_fifo_compact(const float* d_src, float* d_dst, uint64_t stride, const uint32_t* d_drop, const uint32_t* d_keep,
                                  uint32_t n_streams, cudaStream_t st);
// The mixer sum over slots: group g's partial row holds frames of w = slot[g] >> 16 interleaved channels that land on mixer
// channels [o, o + w), o = slot[g] & 0xffff.  out[f * C + j] = +0.0 + every partial row whose slot covers j, in group order.
cudaError_t rb_lanes_launch_sum_slots(const float* d_partial, const uint32_t* d_slot, uint32_t n_groups, uint64_t pstride, uint64_t n_frames,
                                      uint32_t channels, float* d_out, cudaStream_t st);
// rows[r].flags takes the ROW_UNSAFE bit of stream_rows[row_stream[r]] (time-parallel plan: a stream is classified once, its
// segment rows inherit the verdict); row_stream[r] == ~0u (padding) clears it.
cudaError_t rb_lanes_spread_flags(lanes::Row* d_rows, uint32_t n_rows, const uint32_t* d_row_stream, const lanes::Row* d_stream_rows, cudaStream_t st);
// One CTA per stream of d_rows: Row::flags = ROW_UNSAFE when a sample lies outside the exact-reciprocal class.
cudaError_t rb_lanes_launch_classify(lanes::Row* d_rows, uint32_t n_rows, const uint8_t* d_row_channels, cudaStream_t st);
