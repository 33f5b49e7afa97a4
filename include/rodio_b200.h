/*
 * rodio_b200.h — C ABI of the H100-native block DSP path that sits behind rodio's
 * `Source` / `Mixer` / `Player` surface.
 *
 * rodio itself has no FFI; the boundary it exposes for this path is the Rust trait
 * `Source: Iterator<Item = f32>` (reference src/source/mod.rs:179-218) plus the
 * constructors listed per entry point below.  A Rust shim (`bindings/rust/`, shown in
 * INTEGRATION.md) implements `Source` on top of these functions by pulling *blocks*;
 * the per-sample pull model survives only inside that shim.
 *
 * Conventions
 *   - plain C types, caller-owned host memory, no exceptions/panics across the ABI:
 *     every function returns an rb_status (0 = RB_OK); where rodio would panic
 *     (zero rate / zero channels / frequency 0 / clamp(min > max)) the call fails
 *     with RB_ERR_INVALID_ARGUMENT instead.
 *   - thread-compatible: one caller per rb_context / rb_batch at a time.
 *   - all device work is enqueued on the context's CUDA stream; functions that hand
 *     results to the host synchronise that stream before returning, `*_device`
 *     variants do not (use rb_context_sync).
 *   - there is NO CPU fallback: if no CUDA device is usable, rb_context_create fails
 *     with RB_ERR_CUDA and nothing else can be called.
 */
#ifndef RODIO_B200_H
#define RODIO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB_ABI_VERSION 1

typedef int32_t rb_status;
enum {
    RB_OK = 0,
    RB_ERR_INVALID_ARGUMENT = 1, /* NULL pointer, zero rate/channels, bad enum, clamp(min>max) ... */
    RB_ERR_CUDA = 2,             /* CUDA runtime error; text via rb_last_error() */
    RB_ERR_OUT_OF_MEMORY = 3,
    RB_ERR_UNSUPPORTED = 4,      /* a combination the block path does not implement (documented) */
    RB_ERR_UNALIGNED_FRAMES = 5, /* input length is not a whole number of frames */
    RB_ERR_RATIO_OVERFLOW = 6,   /* reduced from*to >= 2^32: rodio's u32 index math would wrap
                                    (reference src/conversions/sample_rate.rs:45-47,:157-158,:173) */
    RB_ERR_NOT_SUPPORTED_SEEK = 7, /* mirrors SeekError::NotSupported (src/source/mod.rs:767-810) */
    RB_ERR_BUFFER_TOO_SMALL = 8,
    RB_ERR_STATE = 9             /* call order violated (e.g. render before upload) */
};

/* Sample formats accepted at the input edge (rows a3 / K8 of SURVEY.md §8).
 * Conversion to f32 follows dasp_sample 0.11.0 `conv` (reference call site
 * src/conversions/sample.rs:42-44; decoder side src/decoder/wav.rs:119-151). */
typedef enum {
    RB_FMT_F32 = 0,
    RB_FMT_I16 = 1,
    RB_FMT_U16 = 2,
    RB_FMT_I8  = 3,
    RB_FMT_U8  = 4,
    RB_FMT_I32 = 5,
    RB_FMT_I24_IN_I32 = 6 /* 24-bit signed value sign-extended in an int32 (dasp I24) */
} rb_sample_format;

/* Effect kinds.  Each replaces one rodio adapter; parameters have the same meaning as
 * the rodio constructor named in the comment. */
typedef enum {
    RB_FX_AMPLIFY = 1,        /* Source::amplify(value)              src/source/mod.rs:307-314, amplify.rs:63-65
                                 f32[0] = factor                                                              */
    RB_FX_SPEED = 2,          /* Source::speed(ratio)                src/source/speed.rs:103-105,:130-133
                                 f32[0] = factor (samples untouched; reported rate changes)                   */
    RB_FX_LOW_PASS = 3,       /* Source::low_pass_with_q(freq, q)    src/source/blt.rs:11-32,:502-560
                                 u32[0] = freq Hz, f32[0] = q (low_pass(freq) == q 0.5)                       */
    RB_FX_HIGH_PASS = 4,      /* Source::high_pass_with_q(freq, q)   src/source/blt.rs:19-40,:523-541         */
    RB_FX_REVERB = 5,         /* Source::reverb(duration, amplitude) src/source/mod.rs:628-634 (mix.rs:43-53, delay.rs:8-16,:68-75)
                                 ns[0] = delay, f32[0] = amplitude                                            */
    RB_FX_AGC = 6,            /* Source::automatic_gain_control(settings) src/source/mod.rs:415-446, agc.rs:183-236,:433-504
                                 f32[0] = target_level, f32[1] = absolute_max_gain, f32[2] = floor (set_floor, agc.rs:386-388)
                                 ns[0] = attack_time, ns[1] = release_time (clamped to 10 s like mod.rs:432-433) */
    RB_FX_LIMIT = 7,          /* Source::limit(LimitSettings)        src/source/limit.rs:94-130,:854-988
                                 f32[0] = threshold dB, f32[1] = knee_width dB, ns[0] = attack, ns[1] = release */
    RB_FX_SPATIAL = 8,        /* Spatial::new(input, emitter, left_ear, right_ear) src/source/spatial.rs:31-69
                                 f32[0..3) emitter, f32[3..6) left ear, f32[6..9) right ear                    */
    RB_FX_CHANNEL_VOLUME = 9, /* ChannelVolume::new(input, volumes)  src/source/channel_volume.rs:30-38,:71-88
                                 u32[0] = number of output channels (1..12), f32[0..n) = volumes               */
    RB_FX_UNIFORM = 10,       /* UniformSourceIterator::new(input, channels, rate) src/source/uniform.rs:33-47
                                 u32[0] = target channels, u32[1] = target sample rate                        */
    RB_FX_DELAY = 11,         /* Source::delay(duration)             src/source/delay.rs:19-29,:68-75
                                 ns[0] = delay                                                                */
    RB_FX_DISTORTION = 12,    /* Source::distortion(gain, threshold) src/source/distortion.rs:8-17,:66-72
                                 f32[0] = gain, f32[1] = threshold (>= 0: clamp(-t, t) panics otherwise)      */
    RB_FX_LINEAR_RAMP = 13,   /* Source::linear_gain_ramp(duration, start, end, clamp_end) src/source/linear_ramp.rs:9-34,:79-104
                                 also fade_in(d) = ramp(d, 0, 1, false) (fadein.rs:8-15) and
                                 fade_out(d) = ramp(d, 1, 0, true) (fadeout.rs:8-15)
                                 ns[0] = duration (> 0), f32[0] = start_gain, f32[1] = end_gain, u32[0] = clamp_end */
    RB_FX_TAKE_DURATION = 14, /* Source::take_duration(duration) [+ set_filter_fadeout] src/source/take.rs:9-26,:34-41,:107-148
                                 ns[0] = duration, u32[0] = 1 when the fade-out filter is set                */
    RB_FX_MIX = 16,           /* Source::mix(other) src/source/mod.rs:253-261, mix.rs:10-53 -- and with it crossfade.rs:10-23:
                                 take_crossfade_with(other, d) = self.take_duration(d) [fade-out filter set] .mix(
                                 other.take_duration(d).fade_in(d)).  u32[0] = index, in the descriptor array of the same
                                 rb_batch_create call, of the SECOND input: a descriptor of its own (PCM or generator, its own
                                 adapters) whose mix_start is RB_MIX_START_CONSUMED -- it is not added to the mixer, one MIX
                                 consumes it.  Both inputs go through UniformSourceIterator::new(_, channels, rate) of the
                                 FIRST input (mix.rs:16-21); s1 + s2 while both run, then whichever is left (mix.rs:43-53).  */
    RB_FX_APPEND = 17,        /* source::from_iter([this buffer, next buffer, ...]) src/source/from_iter.rs:16-127 -- ONE source whose
                                 sample rate and channel count change where one buffer ends and the next begins (a decoder whose
                                 stream changes format, a play list handed to the mixer as one source).  Leading effects only:
                                 effects[0 .. k) = APPEND, each u32[0] = index of the next buffer's descriptor (f32 PCM, no effects of
                                 its own, mix_start = RB_MIX_START_CONSUMED, span_len = n_samples like a SamplesBuffer or 0).  What
                                 follows sees the parameter change the way rodio's adapters do: AMPLIFY; SPEED; LOW/HIGH_PASS keep
                                 their state and recompute the coefficients behind the first sample of the new span
                                 (SpanTracker, src/source/span.rs:66-101 with blt.rs:122-137); AGC recomputes its coefficients and
                                 starts RMS window, peak and gain from scratch (agc.rs:524-548); LIMIT rebuilds its per-channel state
                                 when the channel count changed (limit.rs:651-697); the mixer's UniformSourceIterator re-bootstraps
                                 with the span length and format FromIter reports at that moment (src/source/uniform.rs:50-68,
                                 :83-96).  Other adapters on such a source: RB_ERR_UNSUPPORTED.                                  */
    RB_FX_PAUSE = 18,         /* Pausable (src/source/pausable.rs:8-21,:85-97), what Player::pause / play drive: from inner sample ns[0]
                                 on the adapters in FRONT of this one are not pulled -- a filter there keeps its state -- and ns[1]
                                 whole frames of literal 0.0 are emitted instead (`channels` zeros per frame, wherever in a frame the
                                 pause sets in), then the source carries on where it stopped.  Adapters behind it (the Player's
                                 volume, the mixer's conversion) see the zeros as samples.  ns[0] > the source's length: no effect. */
    RB_FX_SIGNAL = 15         /* SignalGenerator::new(sample_rate, frequency, function).take(n) src/source/signal_generator.rs:107-135
                                 (SineWave / SquareWave / TriangleWave / SawtoothWave = the same at 48 kHz, src/source/sine.rs:23-27):
                                 the SOURCE of the stream instead of uploaded PCM -- only as effects[0] of a descriptor with
                                 n_samples = 0, channels = 1, format f32, span_len = 0 (the generator reports None); generated on
                                 the device: f32 phase accumulation `phase = (phase + 1/(rate/freq)).rem_euclid(1.0)` and, for the
                                 sine, glibc's sinf bit for bit (double-precision polynomial, restated in rb_dsp.cuh).
                                 u32[0] = rb_signal_function, f32[0] = frequency (> 0 and finite: the reference asserts),
                                 ns[0] = n, the number of samples taken from the endless generator.  In a streaming
                                 session ns[0] = UINT64_MAX is the endless generator itself, and the session
                                 generates the samples into the source's FIFO (see rb_session_create) */
} rb_effect_kind;
typedef enum { RB_SIGNAL_SINE = 0, RB_SIGNAL_TRIANGLE = 1, RB_SIGNAL_SQUARE = 2, RB_SIGNAL_SAWTOOTH = 3 } rb_signal_function;
                              /* src/source/signal_generator.rs:40-69 */

typedef struct rb_effect {
    uint32_t kind;     /* rb_effect_kind */
    uint32_t u32[3];
    float    f32[12];
    uint64_t ns[2];    /* std::time::Duration as whole nanoseconds */
} rb_effect;           /* 80 bytes, no padding */

/* One input stream = one rodio source handed to Mixer::add (src/mixer.rs:58-66):
 * an in-memory PCM buffer (SamplesBuffer, src/buffer.rs:40-60) followed by a chain
 * of adapters, applied in array order (effects[0] wraps the buffer first). */
typedef struct rb_stream_desc {
    uint32_t sample_rate;   /* > 0 */
    uint16_t channels;      /* > 0 */
    uint16_t format;        /* rb_sample_format of the uploaded PCM */
    uint64_t n_samples;     /* interleaved samples (frames * channels); must be frame aligned */
    uint32_t span_len;      /* what the source's current_span_len() reports: 0 = None (span-less, e.g.
                               benches/shared.rs:32-34); n_samples for a SamplesBuffer (src/buffer.rs:76-82).
                               UniformSourceIterator re-bootstraps every min(span_len, 32768) samples
                               (src/source/uniform.rs:56,:83-96). */
    uint32_t n_effects;
    const rb_effect* effects;
    uint64_t mix_start;     /* mixer output sample index at which Mixer::add was called; rounded up to
                               the next frame boundary like src/mixer.rs:175-183.  The mixer sums in the
                               order of the add calls: increasing mix_start, ties in array order. */
} rb_stream_desc;

/* mix_start of a descriptor that is the second input of another descriptor's RB_FX_MIX */
#define RB_MIX_START_CONSUMED UINT64_MAX

typedef struct rb_context rb_context;
typedef struct rb_batch rb_batch;

/* rb_batch_create flags */
enum {
    RB_MIX_EXACT_ORDER = 1u << 0,   /* mixer sum strictly sequential in insertion order (bit-exact with
                                       src/mixer.rs:185-198 on one GPU).  resample -> [low/high_pass] -> [amplify] -> mix batches
                                       keep their fused kernel: k_fused_hot hands the running sum of every tile from CTA to
                                       CTA (the whole mix of 4096 sources bit-identical to the reference's, slower than
                                       the default grouping), so does the effect-chain kernel (cfg4), small filter-free
                                       batches use k_lerp_mix in one group; every other chain takes the general path.  Default = ordered partial sums over
                                       contiguous groups of sources (rows of a fused CTA; runs of a short, wide
                                       mix of >= 256 sources) combined in group order: deterministic,
                                       <= 1e-5 * peak, and still the sequential sum for <= one fused stream per SM */
    RB_NO_FUSION = 1u << 1,         /* run one kernel per adapter (debug / cross-check path)                  */
    RB_BIQUAD_TIME_PARALLEL = 1u << 2, /* low/high_pass of a resample -> filter -> [amplify] -> mix batch of mono f32 sources
                                          run time-parallel: the mixer timeline is cut into segments, every source contributes
                                          one row per segment that starts a warm-up in front of it from zero filter state
                                          (arithmetic per sample = the reference's, src/source/blt.rs:558-560).  Taken only for
                                          filters whose f32 rounding noise leaves the 1e-5 * peak tolerance a margin
                                          (noise gain <= 400: cut-offs from about 700 Hz at q = 0.5; most segments are then
                                          bit-identical to the serial run); every other batch is served as without the flag
                                          (exact serial recurrence).  rb_batch_kernel_family tells which: 4 = time-parallel */
    RB_KEEP_STREAM_OUTPUTS = 1u << 3,  /* also keep every stream's post-chain (pre-mix) samples in HBM so
                                          rb_batch_read_stream can return them                                */
    RB_FUSED_LANES = 1u << 4,          /* large batches (chosen automatically from ~128 sources per SM on): serve
                                          [amplify] -> resample -> [low/high_pass] -> [amplify] -> mix, or the chain with the
                                          filter in front of the conversion ([amplify] -> low/high_pass -> [amplify] ->
                                          resample -> [amplify] -> mix: chosen automatically from 32 sources per SM on, no
                                          other fused kernel serves it), of mono (or stereo, into a stereo mixer) f32
                                          sources at or below the mixer's rate -- with the flag also above it, up to twice --
                                          with the lane-per-stream kernel: every stream's samples are bit-identical to the
                                          default path, the mixer sum is a fixed tree over groups of 32 sources
                                          (<= 1e-5 * peak like the default grouping).  Ignored when the batch has
                                          another shape.  Inputs are classified when uploaded: writers through
                                          rb_batch_input_device_ptr ask for the pointer again after rewriting. */
    RB_FUSED_DUO = 1u << 5             /* the large-batch kernels whatever the batch size, the lane-PAIR kernel where the
                                          batch allows it (mono sources below the mixer's rate, neighbours starting in phase:
                                          two sources per lane sharing one index state, mixer sum = pairs, then the tree over
                                          groups of 64), k_fused_lanes elsewhere.  This is what very large batches get without
                                          any flag. */
};

const char* rb_status_string(rb_status s);
/* Thread-local text of the last failure (CUDA error string, offending field ...). */
const char* rb_last_error(void);
uint32_t rb_abi_version(void);

/* One context per GPU: owns the CUDA stream, workspaces and device properties. */
rb_status rb_context_create(int device_ordinal, rb_context** out);
rb_status rb_context_destroy(rb_context* ctx);
rb_status rb_context_sync(rb_context* ctx);
/* The cudaStream_t (as void*) every launch of this context goes to; for callers that
 * time with CUDA events or enqueue a collective behind a render. */
rb_status rb_context_stream(rb_context* ctx, void** cuda_stream_out);
rb_status rb_context_sm_count(rb_context* ctx, int* out);

/* mixer(channels, sample_rate) + Mixer::add for every desc, in array order
 * (src/mixer.rs:25-43,:58-66).  Validates like the reference constructors would
 * panic/accept, computes every stream's output length in closed form and allocates
 * HBM.  `descs[i].effects` are copied. */
rb_status rb_batch_create(rb_context* ctx, uint16_t mixer_channels, uint32_t mixer_sample_rate,
                          const rb_stream_desc* descs, size_t n_streams, uint32_t flags,
                          rb_batch** out);
rb_status rb_batch_destroy(rb_batch* b);

/* Host -> HBM copy of one stream's PCM in the desc's format (the SamplesBuffer::new data). */
rb_status rb_batch_upload(rb_batch* b, size_t stream, const void* pcm, uint64_t n_samples);
/* Upload for many streams laid out back to back in one pinned/pageable host buffer
 * (stream i at element offset sum(n_samples[0..i))). */
rb_status rb_batch_upload_packed(rb_batch* b, const void* pcm, uint64_t total_samples);
/* Device pointer + capacity (in samples of the desc's format) of a stream's input region,
 * for callers that produce PCM on the GPU (bench: inputs resident in HBM). */
rb_status rb_batch_input_device_ptr(rb_batch* b, size_t stream, void** dptr, uint64_t* capacity);

/* Closed-form lengths (samples): the stream after its whole chain incl. the mixer's
 * UniformSourceIterator, and the mixer output. */
rb_status rb_batch_stream_out_len(rb_batch* b, size_t stream, uint64_t* n_samples);
rb_status rb_batch_mix_len(rb_batch* b, uint64_t* n_samples);
/* Number of kernels one rb_batch_render_mix_device enqueues (bench "gpu_launches"). */
rb_status rb_batch_launches_per_render(rb_batch* b, uint32_t* n);
/* Which kernel family serves the batch: -1 = one kernel per adapter (general path), 0 = k_fused_biquad /
 * k_fused_nobiquad, 1 = k_fused_hot, 2 = k_fused_lanes (RB_FUSED_LANES), 3 = k_fused_duo (lane-pair kernel),
 * 4 = time-parallel plan on k_fused_duo (RB_BIQUAD_TIME_PARALLEL).  For tests and bench labels. */
rb_status rb_batch_kernel_family(rb_batch* b, int* family);
/* Summation geometry of the fused mixer sum (src/mixer.rs:185-198 adds the sources sequentially): `rows` consecutive
 * streams (insertion order) form one partial sum -- sequential from +0.0 in k_fused_hot / k_fused_biquad, the fixed
 * 32-lane tree in k_fused_lanes -- and the partial sums are added in order.  0 = the whole mix is one sequential sum
 * (general path, RB_MIX_EXACT_ORDER).  For the parity tests, which rebuild the kernel's documented order from the
 * oracle's per-stream outputs. */
rb_status rb_batch_mix_group(rb_batch* b, uint32_t* rows);
/* ---- multi-GPU: shard the sources over GPUs, one all-reduce for the cross-shard mixer sum (src/mixer.rs:185-198 is the sum
 * being distributed; SURVEY.md 8b / 8e).  NCCL over NVLink, loaded at first use (dlopen libnccl.so.2); RB_ERR_UNSUPPORTED when
 * the box has none.  One process per GPU: rank 0 calls rb_comm_unique_id, hands the 128 bytes to the other ranks by whatever
 * channel the host has, every rank calls rb_comm_init_rank.  One process driving several GPUs: rb_comm_init_all over its
 * contexts.  rb_batch_render_mix_allreduce renders the batch of every LOCAL rank (one per context of the communicator, in
 * order) and sums the mixes over all ranks in place, on the contexts' streams; shards keep the insertion order inside a GPU,
 * the cross-shard association differs from the sequential sum: the fused kernels' tolerance class (<= 1e-5 * peak). ---- */
typedef struct rb_comm rb_comm;
typedef struct { char bytes[128]; } rb_comm_id;
rb_status rb_comm_unique_id(rb_comm_id* id);
rb_status rb_comm_init_rank(rb_context* ctx, int n_ranks, int rank, const rb_comm_id* id, rb_comm** out);
rb_status rb_comm_init_all(rb_context** ctxs, int n_gpus, rb_comm** out);
rb_status rb_comm_destroy(rb_comm* comm);
/* How the mixes travel on this communicator, known after the first rb_batch_render_mix_allreduce: "p2p ..." -- ONE kernel per GPU
 * (k_mix_exchange) forms the shard's mix (adding the fused kernel's partial rows itself), pushes it as (value, tag) pairs into a
 * mailbox in every peer's HBM over NVLink and sums the shards in rank order from +0.0: deterministic and identical on every rank --
 * or "nccl ... (why)": ncclAllReduce, where the ranks cannot map each other's memory (another node, IPC not permitted) or with
 * RB_COMM_NCCL_ONLY=1 in the environment. */
rb_status rb_comm_transport(rb_comm* comm, char* buf, uint64_t cap);
rb_status rb_batch_render_mix_allreduce(rb_batch** batches, int n_local, rb_comm* comm);

/* Algorithmic bytes of one render: 4*sum(in_samples)(or format size) + 4*mix_len. */
rb_status rb_batch_algorithmic_bytes(rb_batch* b, uint64_t* bytes);

/* Pure host query (no device needed): the number of samples MixerSource would pull from this
 * source, i.e. the length of UniformSourceIterator::new(chain, mixer_channels, mixer_rate), plus the
 * channel count / sample rate the chain itself reports (Source::channels / Source::sample_rate).
 * Runs exactly the validation rb_batch_create runs.  Any out pointer may be NULL. */
rb_status rb_stream_plan(const rb_stream_desc* desc, uint16_t mixer_channels, uint32_t mixer_sample_rate,
                         uint64_t* out_len_samples, uint16_t* chain_channels, uint32_t* chain_sample_rate,
                         uint64_t* chain_len_samples);
/* The same for descriptor `stream` of an array: descriptors that name others (RB_FX_MIX, RB_FX_APPEND) need the array. */
rb_status rb_streams_plan(const rb_stream_desc* descs, size_t n_streams, size_t stream, uint16_t mixer_channels, uint32_t mixer_sample_rate,
                          uint64_t* out_len, uint16_t* chain_channels, uint32_t* chain_rate, uint64_t* chain_len);

/* Adapters on the MixerSource itself, in array order: [AMPLIFY] [LIMIT] [AMPLIFY] (each optional, >= 1 effect).
 * rodio: mixer_source.amplify(a).limit(settings).amplify(b) (src/mixer.rs:70-136, src/source/limit.rs).  n_effects = 0 removes it.
 * Records as for a source: RB_FX_AMPLIFY f32[0]; RB_FX_LIMIT f32[0..1], ns[0..1], its coefficients for the mixer's rate and
 * channel count (the mixer's format never changes).  The chain runs over the active runs of the mix as ONE sequence: where
 * MixerSource::next() returns None (no source playing, a later Mixer::add still scheduled) the chain is not pulled, the
 * sample stays 0.0 and the limiter keeps its state.  Every call that hands out the mix (rb_batch_render_mix(_device),
 * rb_batch_mix_device_ptr, rb_batch_read_mix, rb_session_render) then returns the mastered mix; rb_batch_kernel_family and
 * rb_batch_mix_group still describe the sum, rb_batch_launches_per_render counts one launch more (k_master).
 * RB_ERR_UNSUPPORTED: another kind, another order, a second LIMIT or two AMPLIFYs on one side of it.
 * rb_batch_set_master: RB_ERR_UNALIGNED_FRAMES when an active run of the mix ends inside a frame (a chain with a trailing
 * partial frame); rb_batch_render_mix_allreduce refuses a batch with a master chain (RB_ERR_UNSUPPORTED).
 * rb_session_set_master: before the first rendered frame (RB_ERR_STATE after it); the limiter state carries from block to
 * block and travels in the state blob, which only a session with the same master chain accepts. */
rb_status rb_batch_set_master(rb_batch* b, const rb_effect* effects, uint32_t n_effects);

/* Drain the MixerSource (src/mixer.rs:120-136) for the whole batch.
 *   _device: enqueue only; result stays in HBM (rb_batch_mix_device_ptr), no sync.
 *   host   : enqueue, copy `min(mix_len, max_samples)` samples to out_host, sync. */
rb_status rb_batch_render_mix_device(rb_batch* b);
rb_status rb_batch_mix_device_ptr(rb_batch* b, float** dptr);
rb_status rb_batch_render_mix(rb_batch* b, float* out_host, uint64_t max_samples, uint64_t* written);

/* Copy `n_samples` of the rendered mixer output starting at sample `offset` to the host (valid after a
 * render; the block-pulling shim hands these out one block at a time).  Reads past mix_len are clipped;
 * `written` receives the number of samples copied. */
rb_status rb_batch_read_mix(rb_batch* b, uint64_t offset, float* out_host, uint64_t n_samples, uint64_t* written);

/* Per-stream post-chain samples (what MixerSource would pull from that source), for
 * parity tests; needs RB_KEEP_STREAM_OUTPUTS. Valid after a render. */
rb_status rb_batch_read_stream(rb_batch* b, size_t stream, float* out_host, uint64_t max_samples,
                               uint64_t* written);

/* ---- Streaming sessions: sources whose length is not known when they are added --------------------------------
 * rodio pulls MixerSource one sample at a time while decoders produce their sources incrementally
 * (src/mixer.rs:120-136 -> src/source/uniform.rs:78-97 -> src/conversions/sample_rate.rs:131-201 ->
 * src/source/blt.rs:397-410); every adapter keeps its state between pulls.  A session is the block form of that pull:
 * PCM is pushed per source as it arrives, the mixer output is pulled in blocks; the resampler position, the input
 * frames still needed and the filter state carry over from block to block, so ANY split into pushes and renders gives
 * the bytes of a whole-stream rb_batch render with RB_FUSED_LANES (tests/test_lanes_emulator.py::test_session_*).
 * Shape served (RB_ERR_UNSUPPORTED otherwise): a mixer of 1 to 12 channels = mixer(channels, rate) of src/mixer.rs:25-43 (the
 * device's channel count, src/stream.rs); f32 sources of 1 to 12 channels each (a mono mixer: mono sources only), brought to
 * the mixer's count like ChannelCountConverter (src/conversions/channels.rs:57-85): output channel j is input channel j if j < the source's count,
 * channel 0 again if j == 1 and the source is mono, else 0.0 -- a 5.1 source in a stereo mixer keeps its first two channels.
 * A source whose conversion pads channels with 0.0 is refused when the filter behind the conversion has a non-finite
 * coefficient or the gain behind it is not finite (rodio puts NaN on those channels; the session adds nothing there), and
 * rb_session_set_amplify refuses a non-finite factor for it.  Mix order: a source is served as slot rows of at most two
 * mixer channels each (channels 2s, 2s + 1; a mono source in a wider mixer: one row on channels 0 and 1); the rows of all
 * sources, in the caller's order, form classes by rate pair, chain variant and slot; per class groups of 32 rows are summed
 * with the lane kernel's tree, and mixer channel j is +0.0 plus every group whose slot covers j, in class order.  Each source
 * is at its own sample rate (44.1 kHz, 22.05 kHz and 48 kHz sources in one 48 kHz mixer: one kernel launch
 * per rate pair; sources ABOVE the mixer's rate have fast tiles of their own up to a factor of two, the kernel's general per-sample path beyond), effects = [SPEED | AMPLIFY | one LOW_PASS / HIGH_PASS]* UNIFORM(mixer channels, mixer rate)
 * [LOW_PASS | HIGH_PASS] [AMPLIFY] -- the chain of BASELINE cfg3 behind the conversion, and in front of it what a rodio user
 * hands to Mixer::add or appends to a Player (src/player.rs:120-128): any SPEED (it only changes the rate pair), one filter
 * -- it then runs once per INPUT frame with coefficients for the rate its input reports (src/source/blt.rs to_applier) --,
 * one AMPLIFY in front of that filter and one behind it (src/source/amplify.rs:91-95; without a filter: one AMPLIFY).  One
 * filter per source, in front or behind.  In front of all that the chain may begin with a PUSH PROGRAM: any number of LINEAR_RAMP
 * (fade_in / fade_out), TAKE_DURATION and DISTORTION, with AMPLIFY and SPEED among them -- effects [0, p), p one past the last
 * of the three.  Each sample they give is a function of its input sample and its index in the source, so they run as the PCM
 * is pushed, at the rate the SPEEDs in front of each report; the AMPLIFYs behind the program stay the ones rb_session_set_volume
 * and set_amplify change.  A take ends its source at its last frame (padded with 0.0 as take.rs:107-123 does): a push that
 * reaches it is cut there, later pushes are dropped with RB_OK.  Behind a take rodio's conversion restarts every 32768 samples
 * and never pulls the padding; sessions serve takes of one such run in whole frames, or sources at the mixer's rate whose
 * channels pass through or restart on a frame boundary (RB_ERR_UNSUPPORTED otherwise), and no filter behind a take that ends
 * inside a frame; rb_session_create_ex with RB_SESSION_RESTARTS follows those restarts.  Sources of different shapes may share a
 * session (classes of their own); desc.n_samples / span_len are ignored (span_len: unless RB_SESSION_RESTARTS is given),
 * desc.mix_start is the mixer FRAME the source joins at.  Everything below counts frames; PCM is interleaved.
 * GENERATOR SOURCES: a descriptor may begin with RB_FX_SIGNAL under the batch rules (effects[0], n_samples = 0, mono, f32,
 * span_len = 0; the statuses of rb_stream_plan), followed by any chain above (push program, [SPEED | AMPLIFY | one filter]
 * UNIFORM ...).  ns[0] = n: the source ends after n samples; UINT64_MAX: rodio's endless generator, ended by a TAKE_DURATION in
 * its program or by rb_session_skip.  The session generates its samples on the device: a playing or held generator that has not
 * ended holds min(fifo_frames, frames its take still lets through) input frames ahead of its converter, as if they had been pushed
 * -- rb_session_available counts it so and rb_session_render generates what is missing before it plans the block -- so it never
 * holds the mixer up.  It takes no pushes: rb_session_push(_spans) with frames, end_of_stream or marks and rb_session_push_packed
 * (_spans) with a count, end_of_stream or mark for it return RB_ERR_STATE, rb_session_push_silence RB_ERR_UNSUPPORTED (a refused
 * call changes nothing).  Every other call treats it as a pushed source with the same PCM: a session with generators renders the
 * bytes of the same session whose generators are replaced by sources pushed with the generators' samples, for any split.
 * One caller per session; every call returns with the work done (the caller may reuse its buffers). */
typedef struct rb_session rb_session;
/* desc.mix_start of a source that is declared now but handed to the mixer later -- Mixer::add while the mixer is playing
 * (src/mixer.rs:58-66): the source takes pushes at once, renders nothing and holds nobody up until rb_session_start. */
#define RB_SESSION_HELD UINT64_MAX
/* fifo_frames: input frames a source can hold between renders (>= 64); max_block_frames: largest render. */
rb_status rb_session_create(rb_context* ctx, uint16_t mixer_channels, uint32_t mixer_sample_rate, const rb_stream_desc* descs,
                            size_t n_streams, uint32_t fifo_frames, uint32_t max_block_frames, rb_session** out);
/* rb_session_create with flags (0: the same call).  RB_SESSION_RESTARTS: the session restarts the mixer's conversion where rodio
 * does.  UniformSourceIterator converts no source as one run: at every bootstrap it asks current_span_len(), caps the answer at
 * 32768 samples and builds a fresh SampleRateConverter over that many samples, which interpolates inside itself only, emits its
 * last frame raw and starts again at numerator 0 (src/source/uniform.rs:50-68, src/conversions/sample_rate.rs:58-71, :187-199).
 * With the flag desc.span_len means what it means in batches: 0 = None, one run for the whole source; S > 0 = the source reports
 * Some(S) at every bootstrap (a SamplesBuffer: its length), so runs are min(S, 32768) samples until the input ends -- unless the
 * pushes say that the report changes (rb_session_push_spans: a decoder reports the packet it decoded last).  desc.n_samples stays
 * ignored.  A resampled source whose push program holds a TAKE_DURATION restarts every
 * min(samples left in the take, S, 32768) samples, the frames of rb_session_push_silence counted against the run as rodio's Take
 * counts Pausable's zeros: such takes may be longer than one run and may be paused.  Filter state and gains carry across a
 * restart, for any split into pushes and renders.  A source at the mixer's rate keeps no conversion state: its restarts change
 * nothing and are not tracked.  RB_ERR_UNSUPPORTED: a schedule whose runs are not whole frames of the source (span_len not a
 * multiple of its channel count; 3, 5, 6, 7 ... channels under the 32768 cap; a resampled take that ends inside a frame) and runs
 * shorter than two frames.  Such a session writes state blob version 8 when some source has a schedule, version 9 once a push
 * carried span marks. */
#define RB_SESSION_RESTARTS 1u
rb_status rb_session_create_ex(rb_context* ctx, uint16_t mixer_channels, uint32_t mixer_sample_rate, const rb_stream_desc* descs,
                               size_t n_streams, uint32_t fifo_frames, uint32_t max_block_frames, uint32_t flags, rb_session** out);
rb_status rb_session_destroy(rb_session* s);
/* Converter runs of source `stream` that have produced an output so far (1 once a source without a schedule plays; sources at
 * the mixer's rate: see RB_SESSION_RESTARTS), and the launches of the lane kernel's RESTART variants so far: a block in which no
 * source restarts makes none. */
rb_status rb_session_source_runs(rb_session* s, size_t stream, uint64_t* runs_started);
rb_status rb_session_restart_launches(rb_session* s, uint64_t* launches);
/* mixer_source.amplify(a).limit(settings).amplify(b) on the session's output: see rb_batch_set_master. */
rb_status rb_session_set_master(rb_session* s, const rb_effect* effects, uint32_t n_effects);
/* n_frames more frames of source `stream` have arrived; end_of_stream != 0: the source's Iterator::next would return
 * None after them.  RB_ERR_BUFFER_TOO_SMALL when its FIFO cannot take them (render first). */
rb_status rb_session_push(rb_session* s, size_t stream, const float* pcm, uint64_t n_frames, int end_of_stream);
/* The same for every source at once: pcm holds n_frames[0] frames of source 0, then n_frames[1] of source 1, ...;
 * end_of_stream may be NULL.  One host->device copy and one kernel for the whole session. */
rb_status rb_session_push_packed(rb_session* s, const float* pcm, const uint64_t* n_frames, const uint8_t* end_of_stream);
/* What current_span_len() starts to return during a push (RB_SESSION_RESTARTS): after `at` samples of THIS push have been
 * pulled from the source it reports span_len (0 = None).  rodio's decoders report the length of the packet they decoded last
 * (src/decoder/symphonia.rs:199-201), which changes as they play, and UniformSourceIterator asks at every bootstrap before it pulls
 * (src/source/uniform.rs:50-68): a caller that pulls its source sample by sample records the report once before the first pull and
 * after every pull, and passes the changes on as marks. */
typedef struct rb_span_mark {
    uint64_t at;        /* samples of this push the source has yielded when current_span_len() starts to return span_len */
    uint32_t span_len;  /* 0 = None */
    uint32_t pad_;      /* 0 */
} rb_span_mark;
/* rb_session_push / rb_session_push_packed with span marks.  desc.span_len is the report before the first mark; a mark holds until
 * the next one, across pushes (a push without marks, by any of the push calls, leaves the report as it is).  Within a push `at`
 * increases strictly and stays below n_frames * channels; a change seen after the last sample of a push goes at `at` = 0 of the
 * next.  A bootstrap after the source has yielded p samples sees the last mark at or before p (the frames of
 * rb_session_push_silence do not move p: the source is not pulled while paused); its run is min(report, 32768) samples, or less
 * where a take ends first.  A block renders any number of restarts per source in one launch per class.  Sources at the mixer's
 * rate take marks and ignore them.  RB_ERR_STATE: marks on a session created without RB_SESSION_RESTARTS;
 * RB_ERR_INVALID_ARGUMENT: malformed marks; RB_ERR_UNSUPPORTED: a run would begin under a report that is not whole frames of the
 * source or under two frames (also from rb_session_push_silence or a push without marks that reaches such a bootstrap).  A
 * refused push changes nothing.  push_packed_spans: n_marks[i] marks for source i; `marks` holds those of source 0, then 1, ... */
rb_status rb_session_push_spans(rb_session* s, size_t stream, const float* pcm, uint64_t n_frames, const rb_span_mark* marks,
                                uint32_t n_marks, int end_of_stream);
rb_status rb_session_push_packed_spans(rb_session* s, const float* pcm, const uint64_t* n_frames, const uint8_t* end_of_stream,
                                       const uint32_t* n_marks, const rb_span_mark* marks);
/* Player::pause / play for one source: n_frames frames of literal 0.0 behind its push program, what Pausable hands out while
 * paused (src/source/pausable.rs:85-97) -- the program in front is not pulled, so fades and takes stand still.  They take FIFO
 * room like a push (RB_ERR_BUFFER_TOO_SMALL).  RB_ERR_UNSUPPORTED for a source with a filter in front of the conversion:
 * rodio freezes that filter while paused, the session would run it over the zeros. */
rb_status rb_session_push_silence(rb_session* s, size_t stream, uint64_t n_frames);
/* Mixer::add for a source declared with RB_SESSION_HELD: it joins at the mixer frame rendered next (sources join on a frame
 * boundary, src/mixer.rs:175-183).  While no source is playing the session renders nothing and its timeline stands still,
 * as MixerSource::next() returns None (src/mixer.rs:129-135); `ended` stays 0 as long as a held source may still come. */
rb_status rb_session_start(rb_session* s, size_t stream);
/* Queue the held source `stream` behind `predecessor` -- Player::append / queue::queue (src/queue.rs:128-192): it starts on
 * the mixer frame after the predecessor's last, which is known as soon as the predecessor has received its end_of_stream.
 * Each source keeps its own chain and rate pair (the queue's sounds need not share a format).  Sources end on whole frames
 * here, so the queue's padding of a sound that ends mid-frame and its keep-alive silence do not arise. */
rb_status rb_session_follow(rb_session* s, size_t stream, size_t predecessor);
/* Player::skip_one / Player::stop / Skippable::skip for one source (src/player.rs:138-166, :253-276; src/source/skippable.rs): the
 * source's iterator returns None from now on -- its input ends with the last frame the mixer's converter has pulled (what
 * has been pushed beyond is dropped, later pushes are refused), the converter emits what it still owes (the last frame raw,
 * src/conversions/sample_rate.rs:187-199) and the source is finished; a source queued behind it (rb_session_follow) starts right
 * after.  A held source that is skipped never plays. */
rb_status rb_session_skip(rb_session* s, size_t stream);
/* Amplify::set_factor (src/source/amplify.rs:25-29) on the AMPLIFY of a live source's chain: the gain is `factor` from the
 * next rendered block on (a source without an AMPLIFY behaves as amplify(1.0)).  Player::set_volume does the same to its
 * own Amplify every 5 ms of audio (src/player.rs:138-166) -- but that one sits in FRONT of the mixer's resampler
 * (src/player.rs:120-128), while the session's chain amplifies behind it: equal up to the rounding of one multiplication
 * per sample, not bit for bit; an exact Player mirror needs a gain on the taps (not in the session shape yet). */
rb_status rb_session_set_amplify(rb_session* s, size_t stream, float factor);
/* Player::set_volume (src/player.rs:180-186): the Player's Amplify sits IN FRONT of the mixer's conversion, behind the user's
 * source and its filters (src/player.rs:120-128).  Changes that AMPLIFY of the source's chain -- the one in front of the
 * conversion, behind a filter in front if there is one -- for every input frame the converter pulls from the next render on;
 * the (at most two) frames it has pulled already keep the factor they were multiplied with, like Amplify::next
 * (src/source/amplify.rs:91-95).  RB_ERR_STATE when the source was declared without that AMPLIFY. */
rb_status rb_session_set_volume(rb_session* s, size_t stream, float factor);
/* Mixer frames the next render can produce from what has been pushed (an output frame exists once its right input
 * neighbour has arrived, or its source has ended: sample_rate.rs:187-199).  *ended != 0: every source is exhausted
 * and drained -- MixerSource::next() returns None (src/mixer.rs:129-135). */
rb_status rb_session_available(rb_session* s, uint64_t* frames, int* ended);
/* Pull up to max_frames (<= max_block_frames per call) mixer frames into out_host. */
rb_status rb_session_render(rb_session* s, float* out_host, uint64_t max_frames, uint64_t* written, int* ended);
/* Block-to-block state as an opaque blob -- resampler positions, pending input frames, filter state (the
 * rb_batch_get_state / rb_batch_set_state of SURVEY.md 8b): a session of the same shape restored from it, on any
 * context, continues bit-identically.  buf == NULL: only *size is returned.  One record per slot row; a session whose every
 * source is one row carrying all of its channels (mono and stereo mixers, mono sources in any mixer) writes version 5, any
 * other layout version 6 with a layout record per row; a session with push programs writes version 7, which adds the program
 * frames each source has consumed and the programs; a session with restart schedules writes version 8, which adds the converter
 * run of each source; a session with generator sources writes version 10: the blob it would otherwise write, then one record per
 * generator (its phase, the samples it generated).  A blob of another shape, schedule, layout, master chain, program or generator
 * set: RB_ERR_INVALID_ARGUMENT. */
rb_status rb_session_get_state(rb_session* s, void* buf, uint64_t cap, uint64_t* size);
rb_status rb_session_set_state(rb_session* s, const void* buf, uint64_t size);

/* Stand-alone conversions (rows a1..a3 of SURVEY.md §8) on host buffers: H2D, one kernel, D2H.
 *   rb_convert_sample_rate   = SampleRateConverter::new(input, from, to, channels).collect()
 *                              (src/conversions/sample_rate.rs:52-201)
 *   rb_convert_channels      = ChannelCountConverter::new(input, from, to).collect()
 *                              (src/conversions/channels.rs:28,:57-85)
 *   rb_convert_samples       = SampleTypeConverter<_, O>::new(input).collect()
 *                              (src/conversions/sample.rs:14,:42-44)
 * `*_len` query helpers give the exact output length first. */
rb_status rb_sample_rate_out_len(uint64_t n_in, uint32_t from, uint32_t to, uint16_t channels, uint64_t* n_out);
rb_status rb_convert_sample_rate(rb_context* ctx, const float* in, uint64_t n_in, uint32_t from, uint32_t to,
                                 uint16_t channels, float* out, uint64_t cap, uint64_t* n_out);
rb_status rb_channels_out_len(uint64_t n_in, uint16_t from, uint16_t to, uint64_t* n_out);
rb_status rb_convert_channels(rb_context* ctx, const float* in, uint64_t n_in, uint16_t from, uint16_t to,
                              float* out, uint64_t cap, uint64_t* n_out);
rb_status rb_convert_samples(rb_context* ctx, const void* in, rb_sample_format in_fmt, void* out,
                             rb_sample_format out_fmt, uint64_t n);

/* Host-side helpers that mirror rodio's pure functions bit for bit (used by the shim so
 * reported metadata matches):
 *   rb_speed_sample_rate  = Speed::sample_rate()            src/source/speed.rs:130-133
 *   rb_delay_samples      = delay::remaining_samples()      src/source/delay.rs:8-16
 *   rb_db_to_linear / rb_linear_to_db                       src/math.rs:52-56,:87-90
 *   rb_spatial_volumes    = Spatial::set_positions()        src/source/spatial.rs:48-69 */
uint32_t rb_speed_sample_rate(uint32_t input_rate, float factor);
uint64_t rb_delay_samples(uint64_t delay_ns, uint32_t sample_rate, uint16_t channels);
float rb_db_to_linear(float decibels);
float rb_linear_to_db(float linear);
void rb_spatial_volumes(const float emitter[3], const float left_ear[3], const float right_ear[3],
                        float out_volumes[2]);

/* ---- WAV ingest (host only; src/decoder/wav.rs:119-151 reads 8 / 16 / 24 / 32-bit integer and 32-bit float PCM and hands
 * every sample to dasp's to_sample()): rb_wav_parse finds the format and the sample data inside a RIFF/WAVE image so that the
 * bytes of the `.wav` files under assets/ go to HBM as they are (rb_batch_upload with `format`) and are converted on the device by the same
 * rules (8-bit WAV is unsigned: RB_FMT_U8 = hound's i8 after its -128).  24-bit samples are packed in 3 bytes: `format` is then
 * RB_FMT_I24_IN_I32 and `packed24` is set -- widen them with rb_wav_unpack24 first. ---- */
typedef struct rb_wav_info {
    uint32_t sample_rate;
    uint16_t channels;
    uint16_t bits_per_sample;
    uint16_t format;        /* rb_sample_format of the samples (after rb_wav_unpack24 when packed24) */
    uint16_t packed24;      /* 1: the data chunk holds 3-byte little-endian samples */
    uint32_t pad_;
    uint64_t data_offset;   /* byte offset of the first sample inside the image */
    uint64_t data_bytes;    /* bytes of sample data present in the image (a truncated file is cut to whole samples) */
    uint64_t n_samples;     /* interleaved samples */
} rb_wav_info;
/* RB_ERR_INVALID_ARGUMENT: not a RIFF/WAVE image or no fmt / data chunk; RB_ERR_UNSUPPORTED: a sample format rodio's decoder
 * does not read either (compressed tags, float widths other than 32, more than 32 integer bits). */
rb_status rb_wav_parse(const void* image, uint64_t image_bytes, rb_wav_info* out);
void rb_wav_unpack24(const void* packed, uint64_t n_samples, int32_t* out_i24_in_i32);

#ifdef __cplusplus
}
#endif
#endif /* RODIO_B200_H */
