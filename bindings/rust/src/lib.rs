//! `impl Source` on top of the C ABI in include/rodio_b200.h.
//!
//! The per-sample pull model of `rodio::Source` (reference src/source/mod.rs:179-218) survives only
//! here: `GpuMixerSource::next()` hands out samples from a block that one `rb_batch_render_mix` call
//! produced on the GPU.  NOT COMPILED in the build image (no Rust toolchain) — reviewed by hand against
//! the header; every `extern "C"` item below is declared 1:1 in include/rodio_b200.h.
#![allow(non_camel_case_types)]
use std::ffi::c_void;
use std::num::NonZero;
use std::time::Duration;

use rodio::source::SeekError;
use rodio::{ChannelCount, Sample, SampleRate, Source};

#[repr(C)]
#[derive(Clone, Copy)]
pub struct rb_effect {
    pub kind: u32,
    pub u32_: [u32; 3],
    pub f32_: [f32; 12],
    pub ns: [u64; 2],
}

#[repr(C)]
pub struct rb_stream_desc {
    pub sample_rate: u32,
    pub channels: u16,
    pub format: u16,
    pub n_samples: u64,
    pub span_len: u32,
    pub n_effects: u32,
    pub effects: *const rb_effect,
    pub mix_start: u64,
}

pub enum rb_context {}
pub enum rb_batch {}

extern "C" {
    fn rb_context_create(device: i32, out: *mut *mut rb_context) -> i32;
    fn rb_context_destroy(ctx: *mut rb_context) -> i32;
    fn rb_batch_create(ctx: *mut rb_context, mixer_channels: u16, mixer_rate: u32, descs: *const rb_stream_desc,
                       n: usize, flags: u32, out: *mut *mut rb_batch) -> i32;
    fn rb_batch_destroy(b: *mut rb_batch) -> i32;
    fn rb_batch_upload(b: *mut rb_batch, stream: usize, pcm: *const c_void, n_samples: u64) -> i32;
    fn rb_batch_mix_len(b: *mut rb_batch, n: *mut u64) -> i32;
    fn rb_batch_render_mix(b: *mut rb_batch, out: *mut f32, max_samples: u64, written: *mut u64) -> i32;
    fn rb_speed_sample_rate(input_rate: u32, factor: f32) -> u32;
    fn rb_batch_mix_device_ptr(b: *mut rb_batch, dptr: *mut *mut f32) -> i32;
    fn rb_batch_read_mix(b: *mut rb_batch, offset: u64, out: *mut f32, n_samples: u64, written: *mut u64) -> i32;
    // multi-GPU (INTEGRATION.md section 5): one process per GPU; rank 0 makes the id, the host hands its 128 bytes to the others
    fn rb_comm_unique_id(id: *mut rb_comm_id) -> i32;
    fn rb_comm_init_rank(ctx: *mut rb_context, n_ranks: i32, rank: i32, id: *const rb_comm_id, out: *mut *mut rb_comm) -> i32;
    fn rb_comm_destroy(comm: *mut rb_comm) -> i32;
    fn rb_comm_transport(comm: *mut rb_comm, buf: *mut std::os::raw::c_char, cap: u64) -> i32;   // "p2p ..." (NVLink peer memory) or "nccl ... (why)"
    fn rb_batch_render_mix_allreduce(batches: *mut *mut rb_batch, n_local: i32, comm: *mut rb_comm) -> i32;
}
#[repr(C)] pub struct rb_comm { _private: [u8; 0] }
#[repr(C)] #[derive(Clone, Copy)] pub struct rb_comm_id { pub bytes: [u8; 128] }

/// This rank's shard of a mixer that is spread over several GPUs: `render()` leaves the sum over ALL shards on every rank
/// (src/mixer.rs:185-198 is the sum being distributed; shards in rank order = the sources' insertion order).
pub struct GpuShard { batch: *mut rb_batch, comm: *mut rb_comm, mix_len: u64 }
impl GpuShard {
    /// `batch`: the rank's contiguous slice of the sources (already uploaded); `id` from rank 0's `rb_comm_unique_id`.
    pub unsafe fn new(ctx: *mut rb_context, batch: *mut rb_batch, n_ranks: i32, rank: i32, id: &rb_comm_id) -> Result<Self, i32> {
        let mut comm = std::ptr::null_mut();
        let st = rb_comm_init_rank(ctx, n_ranks, rank, id, &mut comm);
        if st != 0 { return Err(st); }
        let mut mix_len = 0u64;
        rb_batch_mix_len(batch, &mut mix_len);
        Ok(Self { batch, comm, mix_len })
    }
    /// render + the cross-shard sum (one kernel over NVLink peer memory, or ncclAllReduce), then the mix on the host
    pub fn render(&mut self) -> Result<Vec<Sample>, i32> {
        let mut b = self.batch;
        let st = unsafe { rb_batch_render_mix_allreduce(&mut b, 1, self.comm) };
        if st != 0 { return Err(st); }
        let mut out = vec![0f32; self.mix_len as usize];
        let mut w = 0u64;
        let st = unsafe { rb_batch_read_mix(self.batch, 0, out.as_mut_ptr(), self.mix_len, &mut w) };
        if st != 0 { return Err(st); }
        out.truncate(w as usize);
        Ok(out)
    }
}
impl Drop for GpuShard { fn drop(&mut self) { unsafe { rb_comm_destroy(self.comm); } } }

pub const RB_FX_AMPLIFY: u32 = 1;
pub const RB_FX_SPEED: u32 = 2;
pub const RB_FX_LOW_PASS: u32 = 3;
pub const RB_FX_HIGH_PASS: u32 = 4;
pub const RB_FX_REVERB: u32 = 5;
pub const RB_FX_AGC: u32 = 6;
pub const RB_FX_LIMIT: u32 = 7;
pub const RB_FX_SPATIAL: u32 = 8;
pub const RB_FX_CHANNEL_VOLUME: u32 = 9;
pub const RB_FX_UNIFORM: u32 = 10;
pub const RB_FX_DELAY: u32 = 11;
pub const RB_FX_DISTORTION: u32 = 12;
pub const RB_FX_LINEAR_RAMP: u32 = 13;
pub const RB_FX_TAKE_DURATION: u32 = 14;
pub const RB_FX_SIGNAL: u32 = 15;      // SignalGenerator::new(rate, freq, f).take(n): generated on the device
pub const RB_FX_MIX: u32 = 16;         // Source::mix(other): u32[0] = descriptor index of the second input
pub const RB_FX_APPEND: u32 = 17;      // source::from_iter([self, next, ..]): u32[0] = descriptor index of the next buffer
pub const RB_FX_PAUSE: u32 = 18;       // Pausable with pause()/play() at known positions: ns[0] = inner sample, ns[1] = frames of silence
pub const RB_MIX_START_CONSUMED: u64 = u64::MAX;   // mix_start of a descriptor another descriptor's MIX / APPEND consumes

/// An in-memory source plus the adapters recorded on it (what `SamplesBuffer::new(..).amplify(..)` builds).
pub struct GpuSource {
    pcm: Vec<Sample>,
    channels: ChannelCount,
    sample_rate: SampleRate,
    span_len: u32,
    effects: Vec<rb_effect>,
    reported_rate: SampleRate,
    /// second inputs of `mix` / buffers appended by `from_iter`: descriptors of their own, `others[k]` belongs to the k-th
    /// RB_FX_MIX / RB_FX_APPEND of `effects` (their u32[0] is filled in when the descriptor array is laid out)
    others: Vec<GpuSource>,
}

impl GpuSource {
    /// `SignalGenerator::new(sample_rate, frequency, f).take(n)` (src/source/signal_generator.rs:85-135); function: 0 sine,
    /// 1 triangle, 2 square, 3 sawtooth.  Nothing is uploaded: the samples are generated in HBM (f32 phase accumulation and
    /// glibc's sinf bit for bit, like `f32::sin` on linux-gnu).  `n = u64::MAX` is the endless generator itself: a streaming
    /// session generates it block by block until a `take_duration` in its chain or `rb_session_skip` ends it; it takes no pushes.
    pub fn signal_generator(sample_rate: SampleRate, frequency: f32, function: u32, n: u64) -> Self {
        assert!(frequency > 0.0, "frequency must be greater than zero");        // signal_generator.rs:112
        Self { pcm: vec![], channels: NonZero::new(1).unwrap(), sample_rate, span_len: 0, effects: vec![], reported_rate: sample_rate,
               others: vec![] }
            .push(RB_FX_SIGNAL, [function, 0, 0], &[frequency], [n, 0])
    }
    /// `source::from_iter(buffers)` (src/source/from_iter.rs:16-27): ONE source whose format changes from buffer to buffer; filters
    /// behind it follow the change like `SpanTracker` makes them (state kept, coefficients recomputed), the mixer re-bootstraps.
    pub fn from_iter(mut buffers: Vec<GpuSource>) -> Self {
        let mut head = buffers.remove(0);
        for b in buffers {
            assert!(b.effects.is_empty(), "from_iter takes plain buffers");
            head = head.push(RB_FX_APPEND, [0; 3], &[], [0; 2]);
            head.others.push(b);
        }
        head
    }
    /// `Pausable` (src/source/pausable.rs:85-97) with `pause()` observed after `at_sample` inner samples and `play()` `n_frames` later:
    /// the adapters recorded so far are not pulled in between (a filter keeps its state), whole frames of zeros are emitted
    pub fn pause_at(self, at_sample: u64, n_frames: u64) -> Self { self.push(RB_FX_PAUSE, [0; 3], &[], [at_sample, n_frames]) }
    /// `Source::mix` (src/source/mod.rs:253-261, mix.rs:10-53)
    pub fn mix(mut self, other: GpuSource) -> Self {
        self.others.push(other);
        self.push(RB_FX_MIX, [0; 3], &[], [0; 2])
    }
    /// `Source::take_crossfade_with` (src/source/mod.rs:444-454, crossfade.rs:10-23)
    pub fn take_crossfade_with(self, other: GpuSource, duration: Duration) -> Self {
        self.take_duration(duration, true).mix(other.take_duration(duration, false).linear_gain_ramp(duration, 0.0, 1.0, false))
    }
    /// `SamplesBuffer::new(channels, sample_rate, data)` (src/buffer.rs:40-60)
    pub fn from_samples(channels: ChannelCount, sample_rate: SampleRate, data: Vec<Sample>) -> Self {
        let span_len = data.len().min(u32::MAX as usize) as u32;
        Self { pcm: data, channels, sample_rate, span_len, effects: vec![], reported_rate: sample_rate, others: vec![] }
    }
    fn push(mut self, kind: u32, u: [u32; 3], f: &[f32], ns: [u64; 2]) -> Self {
        let mut f32_ = [0f32; 12];
        f32_[..f.len()].copy_from_slice(f);
        self.effects.push(rb_effect { kind, u32_: u, f32_, ns });
        self
    }
    /// `Source::amplify` (src/source/mod.rs:307-314)
    pub fn amplify(self, value: f32) -> Self { self.push(RB_FX_AMPLIFY, [0; 3], &[value], [0; 2]) }
    /// `Source::speed` (src/source/speed.rs:103-105,:130-133)
    pub fn speed(mut self, ratio: f32) -> Self {
        let r = unsafe { rb_speed_sample_rate(self.reported_rate.get(), ratio) };
        self.reported_rate = NonZero::new(r).expect("minimum is 1");
        self.push(RB_FX_SPEED, [0; 3], &[ratio], [0; 2])
    }
    /// `Source::low_pass` (src/source/mod.rs:686-692)
    pub fn low_pass(self, freq: u32) -> Self { self.push(RB_FX_LOW_PASS, [freq, 0, 0], &[0.5], [0; 2]) }
    /// `Source::high_pass`
    pub fn high_pass(self, freq: u32) -> Self { self.push(RB_FX_HIGH_PASS, [freq, 0, 0], &[0.5], [0; 2]) }
    /// `Source::reverb` (src/source/mod.rs:628-634)
    pub fn reverb(self, duration: Duration, amplitude: f32) -> Self {
        self.push(RB_FX_REVERB, [0; 3], &[amplitude], [duration.as_nanos() as u64, 0])
    }
    /// `Source::delay` (src/source/delay.rs:19-29)
    pub fn delay(self, duration: Duration) -> Self { self.push(RB_FX_DELAY, [0; 3], &[], [duration.as_nanos() as u64, 0]) }
    /// `Source::distortion` (src/source/mod.rs:726-731)
    pub fn distortion(self, gain: f32, threshold: f32) -> Self { self.push(RB_FX_DISTORTION, [0; 3], &[gain, threshold], [0; 2]) }
    /// `Source::linear_gain_ramp` (src/source/mod.rs:534-546); `fade_in` / `fade_out` are the (0,1,false) / (1,0,true) cases
    pub fn linear_gain_ramp(self, duration: Duration, start: f32, end: f32, clamp_end: bool) -> Self {
        self.push(RB_FX_LINEAR_RAMP, [clamp_end as u32, 0, 0], &[start, end], [duration.as_nanos() as u64, 0])
    }
    /// `Source::take_duration` (src/source/take.rs:9-26); `fadeout` = `TakeDuration::set_filter_fadeout`
    pub fn take_duration(self, duration: Duration, fadeout: bool) -> Self {
        self.push(RB_FX_TAKE_DURATION, [fadeout as u32, 0, 0], &[], [duration.as_nanos() as u64, 0])
    }
    /// `Source::automatic_gain_control` (src/source/mod.rs:415-446): target, max gain, floor; attack / release times
    pub fn automatic_gain_control(self, target: f32, attack: Duration, release: Duration, max_gain: f32) -> Self {
        self.push(RB_FX_AGC, [0; 3], &[target, max_gain, 0.0], [attack.as_nanos() as u64, release.as_nanos() as u64])
    }
    /// `Source::limit` (src/source/limit.rs:94-130): threshold dB, knee dB, attack, release
    pub fn limit(self, threshold: f32, knee_width: f32, attack: Duration, release: Duration) -> Self {
        self.push(RB_FX_LIMIT, [0; 3], &[threshold, knee_width], [attack.as_nanos() as u64, release.as_nanos() as u64])
    }
}

/// `mixer::mixer(channels, sample_rate)` (src/mixer.rs:25-43): `add` is infallible like the reference.
pub struct GpuMixer {
    ctx: *mut rb_context,
    channels: ChannelCount,
    sample_rate: SampleRate,
    sources: Vec<(GpuSource, u64)>,
    position: u64,
}

impl GpuMixer {
    pub fn new(channels: ChannelCount, sample_rate: SampleRate) -> Result<Self, i32> {
        let mut ctx = std::ptr::null_mut();
        let st = unsafe { rb_context_create(0, &mut ctx) };
        if st != 0 { return Err(st); }
        Ok(Self { ctx, channels, sample_rate, sources: vec![], position: 0 })
    }
    /// `Mixer::add` (src/mixer.rs:58-66)
    pub fn add(&mut self, source: GpuSource) { self.sources.push((source, self.position)); }

    /// Drain everything added so far into a block-backed `Source`.
    pub fn into_source(mut self) -> Result<GpuMixerSource, i32> {
        // second inputs of mix() and buffers of from_iter() become descriptors of their own behind the sources that were added
        // (mix_start = RB_MIX_START_CONSUMED), breadth first; the adapter that names them gets their index
        let mut i = 0;
        while i < self.sources.len() {
            let others: Vec<GpuSource> = std::mem::take(&mut self.sources[i].0.others);
            let mut k = self.sources.len() as u32;
            for e in self.sources[i].0.effects.iter_mut().filter(|e| e.kind == RB_FX_MIX || e.kind == RB_FX_APPEND) {
                e.u32_[0] = k;
                k += 1;
            }
            self.sources.extend(others.into_iter().map(|o| (o, RB_MIX_START_CONSUMED)));
            i += 1;
        }
        let descs: Vec<rb_stream_desc> = self.sources.iter().map(|(s, start)| rb_stream_desc {
            sample_rate: s.sample_rate.get(), channels: s.channels.get(), format: 0, n_samples: s.pcm.len() as u64,
            span_len: s.span_len, n_effects: s.effects.len() as u32, effects: s.effects.as_ptr(), mix_start: *start,
        }).collect();
        let mut b = std::ptr::null_mut();
        let st = unsafe { rb_batch_create(self.ctx, self.channels.get(), self.sample_rate.get(), descs.as_ptr(),
                                          descs.len(), 0, &mut b) };
        if st != 0 { return Err(st); }
        for (i, (s, _)) in self.sources.iter().enumerate() {
            let st = unsafe { rb_batch_upload(b, i, s.pcm.as_ptr() as *const c_void, s.pcm.len() as u64) };
            if st != 0 { return Err(st); }
        }
        let mut n = 0u64;
        unsafe { rb_batch_mix_len(b, &mut n) };
        let mut block = vec![0f32; n as usize];
        let mut written = 0u64;
        let st = unsafe { rb_batch_render_mix(b, block.as_mut_ptr(), n, &mut written) };
        unsafe { rb_batch_destroy(b); rb_context_destroy(self.ctx); }
        if st != 0 { return Err(st); }
        block.truncate(written as usize);
        Ok(GpuMixerSource { block, pos: 0, channels: self.channels, sample_rate: self.sample_rate })
    }
}

/// `mixer::MixerSource` (src/mixer.rs:70-136) backed by one rendered block.
pub struct GpuMixerSource {
    block: Vec<Sample>,
    pos: usize,
    channels: ChannelCount,
    sample_rate: SampleRate,
}

impl Iterator for GpuMixerSource {
    type Item = Sample;
    #[inline]
    fn next(&mut self) -> Option<Sample> {
        let s = self.block.get(self.pos).copied();
        self.pos += 1;
        s
    }
}

impl Source for GpuMixerSource {
    fn current_span_len(&self) -> Option<usize> { None }               // src/mixer.rs:88-90
    fn channels(&self) -> ChannelCount { self.channels }
    fn sample_rate(&self) -> SampleRate { self.sample_rate }
    fn total_duration(&self) -> Option<Duration> { None }
    fn try_seek(&mut self, _: Duration) -> Result<(), SeekError> {       // src/mixer.rs:109-113
        Err(SeekError::NotSupported { underlying_source: std::any::type_name::<Self>() })
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Streaming: live `Source`s (decoders, microphones) pulled into a GPU session block by block.
// `rb_session_*` is the block form of MixerSource::next (reference src/mixer.rs:120-136): the shim pulls a block of
// samples from every inner rodio `Source` (the only place their per-sample iterators are driven), pushes the blocks,
// and hands the rendered mixer frames out one by one.  State (resampler position, pending frames, filter state) lives
// in the session, so the block size is free -- 10 ms blocks for a cpal callback, whole seconds for offline renders.
pub enum rb_session {}
pub const RB_SESSION_RESTARTS: u32 = 1;
/// What `current_span_len()` starts to return during a push: after `at` samples of the push (0 = None).
#[repr(C)]
#[derive(Clone, Copy)]
pub struct rb_span_mark { pub at: u64, pub span_len: u32, pub pad_: u32 }
#[repr(C)]
pub struct rb_wav_info { pub sample_rate: u32, pub channels: u16, pub bits_per_sample: u16, pub format: u16, pub packed24: u16, pub pad_: u32,
                         pub data_offset: u64, pub data_bytes: u64, pub n_samples: u64 }

extern "C" {
    fn rb_session_create(ctx: *mut rb_context, mixer_channels: u16, mixer_rate: u32, descs: *const rb_stream_desc, n: usize,
                         fifo_frames: u32, max_block_frames: u32, out: *mut *mut rb_session) -> i32;
    /// `rb_session_create` with flags; `RB_SESSION_RESTARTS`: the conversion restarts every min(span_len, 32768) samples and
    /// behind `take_duration`, as `UniformSourceIterator` does.
    pub fn rb_session_create_ex(ctx: *mut rb_context, mixer_channels: u16, mixer_rate: u32, descs: *const rb_stream_desc, n: usize,
                                fifo_frames: u32, max_block_frames: u32, flags: u32, out: *mut *mut rb_session) -> i32;
    pub fn rb_session_source_runs(s: *mut rb_session, stream: usize, runs_started: *mut u64) -> i32;
    pub fn rb_session_restart_launches(s: *mut rb_session, launches: *mut u64) -> i32;
    fn rb_session_destroy(s: *mut rb_session) -> i32;
    fn rb_session_push_packed(s: *mut rb_session, pcm: *const f32, n_frames: *const u64, end_of_stream: *const u8) -> i32;
    fn rb_session_push_silence(s: *mut rb_session, stream: usize, n_frames: u64) -> i32;
    /// `rb_session_push` / `rb_session_push_packed` with span marks (sessions created with `RB_SESSION_RESTARTS`).
    pub fn rb_session_push_spans(s: *mut rb_session, stream: usize, pcm: *const f32, n_frames: u64, marks: *const rb_span_mark,
                                 n_marks: u32, end_of_stream: i32) -> i32;
    fn rb_session_push_packed_spans(s: *mut rb_session, pcm: *const f32, n_frames: *const u64, end_of_stream: *const u8,
                                    n_marks: *const u32, marks: *const rb_span_mark) -> i32;
    fn rb_session_render(s: *mut rb_session, out: *mut f32, max_frames: u64, written: *mut u64, ended: *mut i32) -> i32;
    fn rb_session_follow(s: *mut rb_session, stream: usize, predecessor: usize) -> i32;
    fn rb_session_skip(s: *mut rb_session, stream: usize) -> i32;
    // WAV ingest: where the samples of a RIFF/WAVE image are and in which rb_sample_format (host only)
    fn rb_wav_parse(image: *const c_void, image_bytes: u64, out: *mut rb_wav_info) -> i32;
    fn rb_wav_unpack24(packed: *const c_void, n_samples: u64, out_i24_in_i32: *mut i32);
    fn rb_session_set_volume(s: *mut rb_session, stream: usize, factor: f32) -> i32;
    fn rb_session_get_state(s: *mut rb_session, buf: *mut c_void, cap: u64, size: *mut u64) -> i32;
    fn rb_session_set_state(s: *mut rb_session, buf: *const c_void, size: u64) -> i32;
}

/// `mixer::mixer(1, rate)` whose inputs are arbitrary mono rodio sources of one sample rate, each followed by
/// `UniformSourceIterator::new(_, 1, rate)[.low_pass(f)][.amplify(g)]` on the GPU.
pub struct GpuLiveMixer {
    session: *mut rb_session,
    inputs: Vec<Box<dyn Source + Send>>,   // the sources being pulled (decoders ...)
    done: Vec<bool>,
    block: Vec<f32>,                       // rendered mixer frames not yet handed out
    at: usize,
    pull_frames: usize,                    // input frames pulled per source and refill
    sample_rate: SampleRate,
    ended: bool,
    // `new_following_spans` only: per source, the last report seen and the changes not pushed yet (samples into the next push)
    reports: Option<Vec<Option<usize>>>,
    pending: Vec<Vec<rb_span_mark>>,
}

impl GpuLiveMixer {
    /// A session over `descs` (one mono chain per input, see `rb_session_create`) fed by pulling `inputs`, `pull_frames` samples
    /// per source and refill.  The conversion runs each source as one run.
    pub fn new(ctx: *mut rb_context, descs: &[rb_stream_desc], inputs: Vec<Box<dyn Source + Send>>, pull_frames: usize,
               sample_rate: SampleRate) -> Result<Self, i32> {
        Self::create(ctx, descs, inputs, pull_frames, sample_rate, false)
    }
    /// The same with `RB_SESSION_RESTARTS`: the mixer's conversion restarts where rodio's `UniformSourceIterator` does, for any
    /// source.  The shim records `current_span_len()` once before the first pull and after every pull, and pushes the changes as
    /// span marks (`rb_session_push_packed_spans`) -- a decoder reports the packet it decoded last.
    pub fn new_following_spans(ctx: *mut rb_context, descs: &[rb_stream_desc], inputs: Vec<Box<dyn Source + Send>>, pull_frames: usize,
                               sample_rate: SampleRate) -> Result<Self, i32> {
        Self::create(ctx, descs, inputs, pull_frames, sample_rate, true)
    }
    fn create(ctx: *mut rb_context, descs: &[rb_stream_desc], inputs: Vec<Box<dyn Source + Send>>, pull_frames: usize,
              sample_rate: SampleRate, spans: bool) -> Result<Self, i32> {
        let mut session: *mut rb_session = std::ptr::null_mut();
        let rc = unsafe {
            if spans {
                rb_session_create_ex(ctx, 1, sample_rate.get(), descs.as_ptr(), descs.len(), (4 * pull_frames).max(4096) as u32, 4096,
                                     RB_SESSION_RESTARTS, &mut session)
            } else {
                rb_session_create(ctx, 1, sample_rate.get(), descs.as_ptr(), descs.len(), (4 * pull_frames).max(4096) as u32, 4096, &mut session)
            }
        };
        if rc != 0 { return Err(rc); }
        let n = inputs.len();
        // the report before the first pull goes first: a mark at 0 of the first push
        let reports = if spans { Some(inputs.iter().map(|s| s.current_span_len()).collect::<Vec<_>>()) } else { None };
        let pending = match &reports {
            Some(r) => r.iter().map(|v| vec![rb_span_mark { at: 0, span_len: v.unwrap_or(0) as u32, pad_: 0 }]).collect(),
            None => vec![Vec::new(); n],
        };
        Ok(GpuLiveMixer { session, inputs, done: vec![false; n], block: Vec::new(), at: 0, pull_frames, sample_rate, ended: false, reports,
                          pending })
    }

    /// `Player::pause` of input `stream` for `n_frames` frames: whole frames of 0.0 go to the mixer while the source (and any
    /// fade or take at the front of its chain) is not pulled -- `Pausable` (src/source/pausable.rs).  Returns the rb_status.
    pub fn push_silence(&mut self, stream: usize, n_frames: u64) -> i32 {
        unsafe { rb_session_push_silence(self.session, stream, n_frames) }
    }

    fn refill(&mut self) {
        // pull up to `pull_frames` samples from every live source -- packed: source 0's block, then source 1's, ...
        let mut pcm: Vec<f32> = Vec::with_capacity(self.inputs.len() * self.pull_frames);
        let mut n = vec![0u64; self.inputs.len()];
        let mut eos = vec![0u8; self.inputs.len()];
        let mut marks: Vec<rb_span_mark> = Vec::new();
        let mut n_marks = vec![0u32; self.inputs.len()];
        for (i, src) in self.inputs.iter_mut().enumerate() {
            if self.done[i] { continue; }
            for _ in 0..self.pull_frames {
                match src.next() {
                    Some(s) => { pcm.push(s); n[i] += 1; }
                    None => { self.done[i] = true; eos[i] = 1; break; }
                }
                if let Some(r) = self.reports.as_mut() {      // a change seen after `n[i]` samples of this push
                    let now = src.current_span_len();
                    if now != r[i] {
                        r[i] = now;
                        let m = rb_span_mark { at: n[i], span_len: now.unwrap_or(0) as u32, pad_: 0 };
                        match self.pending[i].last_mut() {
                            Some(last) if last.at == m.at => *last = m,
                            _ => self.pending[i].push(m),
                        }
                    }
                }
            }
            if self.reports.is_some() {   // marks inside this push go now; one after its last sample waits for the next push (at 0)
                let keep: Vec<rb_span_mark> = self.pending[i].iter().filter(|m| m.at >= n[i]).map(|m| rb_span_mark { at: 0, ..*m }).collect();
                for m in self.pending[i].iter().filter(|m| m.at < n[i]) { marks.push(*m); n_marks[i] += 1; }
                self.pending[i] = keep.into_iter().last().into_iter().collect();
            }
        }
        self.block.resize(4096, 0.0);
        let (mut written, mut ended) = (0u64, 0i32);
        unsafe {
            if self.reports.is_some() {
                rb_session_push_packed_spans(self.session, pcm.as_ptr(), n.as_ptr(), eos.as_ptr(), n_marks.as_ptr(), marks.as_ptr());
            } else {
                rb_session_push_packed(self.session, pcm.as_ptr(), n.as_ptr(), eos.as_ptr());
            }
            rb_session_render(self.session, self.block.as_mut_ptr(), 4096, &mut written, &mut ended);
        }
        self.block.truncate(written as usize);
        self.at = 0;
        self.ended = ended != 0;
    }
}

impl Iterator for GpuLiveMixer {
    type Item = Sample;
    fn next(&mut self) -> Option<Sample> {
        while self.at == self.block.len() {
            if self.ended { return None; }                                  // src/mixer.rs:129-135
            self.refill();
        }
        self.at += 1;
        Some(self.block[self.at - 1])
    }
}

impl Source for GpuLiveMixer {
    fn current_span_len(&self) -> Option<usize> { None }
    fn channels(&self) -> ChannelCount { NonZero::new(1).unwrap() }
    fn sample_rate(&self) -> SampleRate { self.sample_rate }
    fn total_duration(&self) -> Option<Duration> { None }
    fn try_seek(&mut self, _: Duration) -> Result<(), SeekError> {
        Err(SeekError::NotSupported { underlying_source: std::any::type_name::<Self>() })
    }
}

impl Drop for GpuLiveMixer {
    fn drop(&mut self) { unsafe { rb_session_destroy(self.session); } }
}

/// The controls of `Player` (reference src/player.rs) on a session.  rodio builds, per appended sound,
/// `speed -> track_position -> pausable -> amplify(volume) -> skippable -> stoppable -> periodic_access(5 ms)` and lets the
/// mixer convert the result (src/player.rs:120-166).  On a session that chain is declared when the sound's slot is created
/// -- `[SPEED] [user effects: AMPLIFY, LOW_PASS ...] AMPLIFY(volume) UNIFORM(mixer)` with `mix_start = RB_SESSION_HELD` -- and
/// the controls become:
///   append      rb_session_follow(slot, previous slot)     the sound starts on the frame after its predecessor's last
///   set_volume  rb_session_set_volume(slot, v)             the Amplify in front of the conversion; frames the converter has
///                                                          pulled already keep their factor, like Amplify::next
///   pause/play  the shim pushes zero frames instead of pulling the source while paused (Pausable emits whole frames of
///               zeros in front of the converter, src/source/pausable.rs:85-97)
///   stop/skip   end_of_stream for the slot (Stoppable / Skippable end the inner iterator, the queue moves on)
///   set_speed   read when the sound is appended (Speed only changes the rate the source reports, src/source/speed.rs:130-133)
pub struct GpuPlayer<'a> {
    mixer: &'a mut GpuLiveMixer,
    slots: Vec<usize>,         // session slots of the sounds appended so far, in order
    paused: bool,
}

impl<'a> GpuPlayer<'a> {
    pub fn append_slot(&mut self, slot: usize) {
        if let Some(&prev) = self.slots.last() { unsafe { rb_session_follow(self.mixer.session, slot, prev); } }
        self.slots.push(slot);
    }
    pub fn set_volume(&mut self, value: f32) {
        for &slot in &self.slots { unsafe { rb_session_set_volume(self.mixer.session, slot, value); } }
    }
    pub fn pause(&mut self) { self.paused = true; }     // GpuLiveMixer::refill pushes zeros for these slots while set
    pub fn play(&mut self) { self.paused = false; }
    pub fn is_paused(&self) -> bool { self.paused }
}
