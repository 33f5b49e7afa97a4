"""Host-side mirror of rodio's `Source` / `Mixer` surface for the H100 block path.

Names, argument meaning and error behaviour follow the reference (file:line in each docstring);
where rodio panics this raises ValueError / RodioB200Error.  Nothing here touches samples on the
CPU: a `Source` is a PCM buffer plus a recorded adapter chain, and `MixerSource` drains it through
the C ABI (include/rodio_b200.h) on the GPU.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from fractions import Fraction
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _capi as capi
from ._capi import check, lib

_NP_OF_FMT = {
    capi.RB_FMT_F32: np.float32, capi.RB_FMT_I16: np.int16, capi.RB_FMT_U16: np.uint16,
    capi.RB_FMT_I8: np.int8, capi.RB_FMT_U8: np.uint8, capi.RB_FMT_I32: np.int32,
}
_FMT_OF_NP = {np.dtype(v): k for k, v in _NP_OF_FMT.items()}


# ---------------------------------------------------------------------------------------------
# std::time::Duration as whole nanoseconds
# ---------------------------------------------------------------------------------------------
class Duration(int):
    """std::time::Duration; the value is whole nanoseconds."""

    @staticmethod
    def from_secs(s: int) -> "Duration":
        return Duration(int(s) * 1_000_000_000)

    @staticmethod
    def from_millis(ms: int) -> "Duration":
        return Duration(int(ms) * 1_000_000)

    @staticmethod
    def from_micros(us: int) -> "Duration":
        return Duration(int(us) * 1_000)

    @staticmethod
    def from_nanos(ns: int) -> "Duration":
        return Duration(int(ns))

    @staticmethod
    def from_secs_f32(secs: float) -> "Duration":
        """Duration::from_secs_f32: the f32 value, rounded to the nearest nanosecond."""
        v = Fraction(float(np.float32(secs)))
        if v < 0:
            raise ValueError("negative Duration (Duration::from_secs_f32 panics)")
        ns = v * 1_000_000_000
        fl = ns.numerator // ns.denominator
        rem = ns - fl
        if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
            fl += 1
        return Duration(fl)


# ---------------------------------------------------------------------------------------------
# effect records (one per rodio adapter)
# ---------------------------------------------------------------------------------------------
@dataclass
class Effect:
    kind: int
    u32: Tuple[int, int, int] = (0, 0, 0)
    f32: Tuple[float, ...] = (0.0,) * 12
    ns: Tuple[int, int] = (0, 0)
    other: Optional["Source"] = None      # RB_FX_MIX: the second input (packed as a descriptor of its own, u32[0] = its index)

    @staticmethod
    def make(kind, u32=(), f32=(), ns=(), other=None):
        u = tuple(int(x) for x in u32) + (0,) * (3 - len(u32))
        f = tuple(float(x) for x in f32) + (0.0,) * (12 - len(f32))
        n = tuple(int(x) for x in ns) + (0,) * (2 - len(ns))
        return Effect(kind, u, f, n, other)


@dataclass
class AutomaticGainControlSettings:
    """src/source/agc.rs:57-82 (defaults :73-82)."""
    target_level: float = 1.0
    attack_time: int = Duration.from_secs(4)
    release_time: int = Duration.from_secs(0)
    absolute_max_gain: float = 7.0
    floor: float = 0.0   # AutomaticGainControl::set_floor (agc.rs:386-388); 0.0 == None


@dataclass
class LimitSettings:
    """src/source/limit.rs:209-248 and the presets :284-438."""
    threshold: float = -1.0
    knee_width: float = 4.0
    attack: int = Duration.from_millis(5)
    release: int = Duration.from_millis(100)

    @staticmethod
    def default() -> "LimitSettings":
        return LimitSettings()

    @staticmethod
    def dynamic_content() -> "LimitSettings":
        return LimitSettings(threshold=-3.0, knee_width=6.0)

    @staticmethod
    def broadcast() -> "LimitSettings":
        return LimitSettings(knee_width=2.0, attack=Duration.from_millis(3), release=Duration.from_millis(50))

    @staticmethod
    def mastering() -> "LimitSettings":
        return LimitSettings(-0.5, 1.0, Duration.from_millis(1), Duration.from_millis(200))

    @staticmethod
    def live_performance() -> "LimitSettings":
        return LimitSettings(-2.0, 3.0, Duration.from_micros(500), Duration.from_millis(30))

    @staticmethod
    def gaming() -> "LimitSettings":
        return LimitSettings(-3.0, 3.0, Duration.from_millis(2), Duration.from_millis(75))

    def with_threshold(self, v):
        return LimitSettings(float(v), self.knee_width, self.attack, self.release)

    def with_knee_width(self, v):
        return LimitSettings(self.threshold, float(v), self.attack, self.release)

    def with_attack(self, v):
        return LimitSettings(self.threshold, self.knee_width, int(v), self.release)

    def with_release(self, v):
        return LimitSettings(self.threshold, self.knee_width, self.attack, int(v))


# ---------------------------------------------------------------------------------------------
# trait Source (src/source/mod.rs:179-759): PCM + recorded adapter chain
# ---------------------------------------------------------------------------------------------
def amplify_effect(value: float) -> Effect:
    """The record of Source::amplify / MixerSource::amplify (src/source/amplify.rs:63-65)."""
    return Effect.make(capi.RB_FX_AMPLIFY, f32=[value])


def limit_effect(settings: Optional[LimitSettings] = None) -> Effect:
    """The record of Source::limit / MixerSource::limit (src/source/limit.rs:94-130)."""
    s = settings or LimitSettings()
    return Effect.make(capi.RB_FX_LIMIT, f32=[s.threshold, s.knee_width], ns=[s.attack, s.release])


def effect_records(effects: Sequence[Effect]):
    """The rb_effect array of a master chain (adapters on the MixerSource: rb_batch_set_master / rb_session_set_master)."""
    fx = (capi.rb_effect * max(1, len(effects)))()
    for j, e in enumerate(effects):
        fx[j].kind = e.kind
        for k in range(3):
            fx[j].u32[k] = e.u32[k]
        for k in range(12):
            fx[j].f32[k] = e.f32[k]
        for k in range(2):
            fx[j].ns[k] = e.ns[k]
    return fx


class Source:
    def __init__(self, pcm: np.ndarray, channels: int, sample_rate: int, span_len: int,
                 effects: Optional[List[Effect]] = None, cur_channels: Optional[int] = None,
                 cur_rate: Optional[int] = None):
        if channels <= 0 or sample_rate <= 0:
            raise ValueError("channels and sample_rate must be non-zero (NonZero in rodio)")
        pcm = np.ascontiguousarray(pcm)
        if pcm.dtype not in _FMT_OF_NP:
            pcm = pcm.astype(np.float32)
        self.pcm = pcm.reshape(-1)
        self.base_channels = int(channels)
        self.base_rate = int(sample_rate)
        self.span_len = int(span_len)
        self.effects: List[Effect] = list(effects or [])
        self._channels = int(cur_channels if cur_channels is not None else channels)
        self._rate = int(cur_rate if cur_rate is not None else sample_rate)
        self.fmt_override: Optional[int] = None     # rb_sample_format the dtype cannot tell (24-bit values in int32)

    # -- metadata the trait reports --------------------------------------------------------
    def channels(self) -> int:
        return self._channels

    def sample_rate(self) -> int:
        return self._rate

    def _with(self, e: Effect, channels=None, rate=None) -> "Source":
        out = Source(self.pcm, self.base_channels, self.base_rate, self.span_len, self.effects + [e],
                     channels if channels is not None else self._channels,
                     rate if rate is not None else self._rate)
        out.fmt_override = self.fmt_override
        return out

    # -- adapters ---------------------------------------------------------------------------
    def amplify(self, value: float) -> "Source":
        """Source::amplify — src/source/mod.rs:307-314."""
        return self._with(amplify_effect(value))

    def amplify_decibel(self, value: float) -> "Source":
        """Source::amplify_decibel — src/source/mod.rs:316-323 (math::db_to_linear)."""
        return self.amplify(lib().rb_db_to_linear(C.c_float(value)))

    def amplify_normalized(self, value: float) -> "Source":
        """Source::amplify_normalized — src/source/mod.rs:325-349."""
        v = np.float32(min(max(np.float32(value), np.float32(0.0)), np.float32(1.0)))
        amp = np.float32(np.exp(np.float32(6.9077554) * v, dtype=np.float32) / np.float32(1000.0))
        if v < np.float32(0.1):
            amp = np.float32(amp * np.float32(v * np.float32(10.0)))
        return self.amplify(float(amp))

    def speed(self, ratio: float) -> "Source":
        """Source::speed — src/source/speed.rs:103-105,:130-133 (samples untouched, rate rescaled)."""
        new_rate = lib().rb_speed_sample_rate(self._rate, C.c_float(ratio))
        return self._with(Effect.make(capi.RB_FX_SPEED, f32=[ratio]), rate=new_rate)

    def low_pass(self, freq: int) -> "Source":
        """Source::low_pass — src/source/mod.rs:686-692 (q = 0.5, blt.rs:11-16)."""
        return self.low_pass_with_q(freq, 0.5)

    def low_pass_with_q(self, freq: int, q: float) -> "Source":
        return self._with(Effect.make(capi.RB_FX_LOW_PASS, u32=[freq], f32=[q]))

    def high_pass(self, freq: int) -> "Source":
        return self.high_pass_with_q(freq, 0.5)

    def high_pass_with_q(self, freq: int, q: float) -> "Source":
        return self._with(Effect.make(capi.RB_FX_HIGH_PASS, u32=[freq], f32=[q]))

    def reverb(self, duration: int, amplitude: float) -> "Source":
        """Source::reverb — src/source/mod.rs:628-634."""
        return self._with(Effect.make(capi.RB_FX_REVERB, f32=[amplitude], ns=[duration]))

    def delay(self, duration: int) -> "Source":
        """Source::delay — src/source/delay.rs:19-29."""
        return self._with(Effect.make(capi.RB_FX_DELAY, ns=[duration]))

    def distortion(self, gain: float, threshold: float) -> "Source":
        """Source::distortion — src/source/mod.rs:726-731 (distortion.rs:66-72)."""
        return self._with(Effect.make(capi.RB_FX_DISTORTION, f32=[gain, threshold]))

    def linear_gain_ramp(self, duration: int, start_value: float, end_value: float, clamp_end: bool) -> "Source":
        """Source::linear_gain_ramp — src/source/mod.rs:534-546 (linear_ramp.rs:79-104)."""
        if int(duration) == 0:
            raise ValueError("duration must be greater than zero (linear_ramp.rs:19)")
        return self._with(Effect.make(capi.RB_FX_LINEAR_RAMP, u32=[1 if clamp_end else 0], f32=[start_value, end_value],
                                      ns=[duration]))

    def fade_in(self, duration: int) -> "Source":
        """Source::fade_in — src/source/fadein.rs:8-15."""
        return self.linear_gain_ramp(duration, 0.0, 1.0, False)

    def fade_out(self, duration: int) -> "Source":
        """Source::fade_out — src/source/fadeout.rs:8-15."""
        return self.linear_gain_ramp(duration, 1.0, 0.0, True)

    def take_duration(self, duration: int, filter_fadeout: bool = False) -> "Source":
        """Source::take_duration (+ TakeDuration::set_filter_fadeout) — src/source/take.rs:9-26,:89-96."""
        return self._with(Effect.make(capi.RB_FX_TAKE_DURATION, u32=[1 if filter_fadeout else 0], ns=[duration]))

    def pause_at(self, at_sample: int, n_frames: int) -> "Source":
        """Pausable (src/source/pausable.rs:85-97) with Player::pause / play scripted: when `at_sample` samples have been pulled
        from this source it stops being pulled -- filters in front keep their state -- and `n_frames` whole frames of zeros follow,
        then it carries on."""
        return self._with(Effect.make(capi.RB_FX_PAUSE, ns=[int(at_sample), int(n_frames)]))

    def mix(self, other: "Source") -> "Source":
        """Source::mix(other) -- src/source/mod.rs:253-261, mix.rs:10-53: both inputs converted to THIS source's channels and rate,
        summed while both run, then whichever is left."""
        return self._with(Effect.make(capi.RB_FX_MIX, other=other))

    def take_crossfade_with(self, other: "Source", duration: int) -> "Source":
        """Source::take_crossfade_with -- src/source/mod.rs:444-454 = crossfade::crossfade (crossfade.rs:10-23)."""
        return self.take_duration(duration, filter_fadeout=True).mix(other.take_duration(duration).fade_in(duration))

    def automatic_gain_control(self, settings: Optional[AutomaticGainControlSettings] = None) -> "Source":
        """Source::automatic_gain_control — src/source/mod.rs:415-446."""
        s = settings or AutomaticGainControlSettings()
        return self._with(Effect.make(capi.RB_FX_AGC, f32=[s.target_level, s.absolute_max_gain, s.floor],
                                      ns=[s.attack_time, s.release_time]))

    def limit(self, settings: Optional[LimitSettings] = None) -> "Source":
        """Source::limit — src/source/limit.rs:94-130."""
        return self._with(limit_effect(settings))

    # -- draining ----------------------------------------------------------------------------
    def collect(self, ctx: Optional["Context"] = None) -> np.ndarray:
        """`.collect::<Vec<f32>>()` of this source (chain only, no mixer conversion)."""
        u = self if self.effects and self.effects[-1].kind == capi.RB_FX_UNIFORM else self
        b = Batch([u], u.channels(), u.sample_rate(), flags=capi.RB_KEEP_STREAM_OUTPUTS | capi.RB_NO_FUSION, ctx=ctx)
        try:
            b.upload_all()
            b.render_mix_device()
            return b.read_stream(0)
        finally:
            b.close()


class SamplesBuffer(Source):
    """buffer::SamplesBuffer::new(channels, sample_rate, data) — src/buffer.rs:40-60.
    `current_span_len()` reports the whole buffer (src/buffer.rs:76-82)."""

    def __init__(self, channels: int, sample_rate: int, data):
        data = np.asarray(data)
        if data.dtype not in _FMT_OF_NP:
            data = data.astype(np.float32)
        super().__init__(data, channels, sample_rate, span_len=min(int(data.size), 0xFFFFFFFF))


class TestSource(Source):
    """benches/shared.rs:7-50 TestSource: a Vec-backed source whose span is `None` (forever)."""
    __test__ = False

    def __init__(self, samples, channels: int, sample_rate: int):
        super().__init__(np.asarray(samples), channels, sample_rate, span_len=0)


def from_iter(sources: Sequence[Source]) -> Source:
    """source::from_iter(sources) -- src/source/from_iter.rs:16-27: the buffers played one after the other as ONE source whose
    sample rate and channel count change where one ends and the next begins (RB_FX_APPEND).  The parts are plain f32 buffers
    (SamplesBuffer or TestSource, no adapters of their own); adapters go on the result."""
    parts = list(sources)
    if not parts:
        raise ValueError("from_iter of nothing")
    for p in parts:
        if p.effects or p.pcm.dtype != np.float32:
            raise ValueError("from_iter takes plain f32 buffers")
    head = parts[0]
    fx = [Effect.make(capi.RB_FX_APPEND, other=o) for o in parts[1:]]
    return Source(head.pcm, head.base_channels, head.base_rate, head.span_len, fx)


class Function:
    """source::Function -- src/source/signal_generator.rs:40-49."""
    Sine, Triangle, Square, Sawtooth = capi.RB_SIGNAL_SINE, capi.RB_SIGNAL_TRIANGLE, capi.RB_SIGNAL_SQUARE, capi.RB_SIGNAL_SAWTOOTH


ENDLESS = 2**64 - 1     # ns[0] of RB_FX_SIGNAL: the generator never ends by itself


class SignalGenerator:
    """source::SignalGenerator::new(sample_rate, frequency, function) -- src/source/signal_generator.rs:85-99: an endless mono
    source; `.take(n)` (Iterator::take, what the reference's tests and examples bound it with) gives the Source that is handed
    to the mixer.  The samples are generated on the device (RB_FX_SIGNAL): nothing is uploaded.
    The Source adapters apply to the endless generator, as in rodio: `SineWave(740.0).amplify(0.1).take_duration(d)` -- a
    streaming Session plays such a source until its take_duration ends it or Session.skip stops it."""

    _ADAPTERS = frozenset(n for n in vars(Source) if not n.startswith("_") and n not in ("channels", "sample_rate", "collect"))

    def __init__(self, sample_rate: int, frequency: float, f: int = Function.Sine):
        if not float(np.float32(frequency)) > 0.0:
            raise ValueError("frequency must be greater than zero (signal_generator.rs:112)")
        self.rate, self.frequency, self.function = int(sample_rate), float(np.float32(frequency)), int(f)

    def channels(self) -> int:
        return 1

    def sample_rate(self) -> int:
        return self.rate

    def take(self, n: int) -> Source:
        e = Effect.make(capi.RB_FX_SIGNAL, u32=[self.function], f32=[self.frequency], ns=[int(n)])
        return Source(np.zeros(0, dtype=np.float32), 1, self.rate, 0, [e])

    def endless(self) -> Source:
        """The generator itself as a Source (ns[0] = ENDLESS)."""
        return self.take(ENDLESS)

    def __getattr__(self, name):
        if name in SignalGenerator._ADAPTERS:
            return getattr(self.endless(), name)
        raise AttributeError(name)


def SineWave(freq: float) -> SignalGenerator:
    """source::SineWave::new(freq): 48 kHz mono -- src/source/sine.rs:23-27."""
    return SignalGenerator(48000, freq, Function.Sine)


def SquareWave(freq: float) -> SignalGenerator:
    return SignalGenerator(48000, freq, Function.Square)


def TriangleWave(freq: float) -> SignalGenerator:
    return SignalGenerator(48000, freq, Function.Triangle)


def SawtoothWave(freq: float) -> SignalGenerator:
    return SignalGenerator(48000, freq, Function.Sawtooth)


class WavInfo(C.Structure):
    _fields_ = [("sample_rate", C.c_uint32), ("channels", C.c_uint16), ("bits_per_sample", C.c_uint16), ("format", C.c_uint16),
                ("packed24", C.c_uint16), ("pad_", C.c_uint32), ("data_offset", C.c_uint64), ("data_bytes", C.c_uint64),
                ("n_samples", C.c_uint64)]


def wav_source(image: bytes) -> Source:
    """Decoder::new_wav(..) as far as this path goes (src/decoder/wav.rs:119-151): the samples of a RIFF/WAVE image in their own
    format -- s16, u8, s32, f32, or 24-bit widened to i24-in-i32 -- as a Source; the conversion to f32 happens on the device by
    dasp's rules (rb_wav_parse / rb_wav_unpack24)."""
    info = WavInfo()
    buf = (C.c_char * len(image)).from_buffer_copy(image)
    check(lib().rb_wav_parse(buf, len(image), C.byref(info)), "rb_wav_parse")
    raw = np.frombuffer(image, dtype=np.uint8, count=info.data_bytes, offset=info.data_offset)
    if info.packed24:
        out = np.empty(info.n_samples, dtype=np.int32)
        lib().rb_wav_unpack24(raw.ctypes.data_as(C.c_void_p), info.n_samples, out.ctypes.data_as(C.c_void_p))
        src = Source(out, info.channels, info.sample_rate, span_len=0)
        src.fmt_override = capi.RB_FMT_I24_IN_I32
        return src
    dt = {capi.RB_FMT_F32: np.float32, capi.RB_FMT_I16: np.int16, capi.RB_FMT_U8: np.uint8, capi.RB_FMT_I32: np.int32}[info.format]
    return Source(raw.view(dt).copy(), info.channels, info.sample_rate, span_len=0)


def ChannelVolume(input: Source, channel_volumes: Sequence[float]) -> Source:
    """source::ChannelVolume::new(input, volumes) — src/source/channel_volume.rs:30-38."""
    vols = [float(v) for v in channel_volumes]
    if not 1 <= len(vols) <= 12:
        raise ValueError("1..12 channel volumes")
    return input._with(Effect.make(capi.RB_FX_CHANNEL_VOLUME, u32=[len(vols)], f32=vols), channels=len(vols))


def Spatial(input: Source, emitter_position, left_ear, right_ear) -> Source:
    """source::Spatial::new(input, emitter, left_ear, right_ear) — src/source/spatial.rs:31-45."""
    f = [float(x) for x in list(emitter_position) + list(left_ear) + list(right_ear)]
    return input._with(Effect.make(capi.RB_FX_SPATIAL, f32=f), channels=2)


def UniformSourceIterator(input: Source, target_channels: int, target_sample_rate: int) -> Source:
    """source::UniformSourceIterator::new(input, channels, rate) — src/source/uniform.rs:33-47."""
    if target_channels <= 0 or target_sample_rate <= 0:
        raise ValueError("target channels / rate must be non-zero")
    if isinstance(input, SignalGenerator):
        input = input.endless()
    return input._with(Effect.make(capi.RB_FX_UNIFORM, u32=[target_channels, target_sample_rate]),
                       channels=target_channels, rate=target_sample_rate)


# ---------------------------------------------------------------------------------------------
# context / batch (thin RAII over the C ABI)
# ---------------------------------------------------------------------------------------------
class Context:
    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        check(lib().rb_context_create(device, C.byref(self._h)), "rb_context_create")
        self.device = device

    def sync(self):
        check(lib().rb_context_sync(self._h), "rb_context_sync")

    @property
    def cuda_stream(self) -> int:
        p = C.c_void_p()
        check(lib().rb_context_stream(self._h, C.byref(p)), "rb_context_stream")
        return p.value or 0

    @property
    def sm_count(self) -> int:
        n = C.c_int()
        check(lib().rb_context_sm_count(self._h, C.byref(n)), "rb_context_sm_count")
        return n.value

    def close(self):
        if self._h:
            lib().rb_context_destroy(self._h)
            self._h = C.c_void_p()


class Comm:
    """The cross-shard mixer sum (include/rodio_b200.h rb_comm_*): NCCL, called by the library on the context's stream.
    One process per GPU: rank 0 calls Comm.unique_id() and hands the bytes to the others (torchrun: broadcast_object_list),
    every rank builds Comm(ctx, n_ranks, rank, id).  One process, several GPUs: Comm.all([ctx0, ctx1, ...])."""

    def __init__(self, ctx: Context, n_ranks: int, rank: int, id_bytes: bytes):
        assert len(id_bytes) == 128
        self._h = C.c_void_p()
        self._ctxs = [ctx]
        buf = (C.c_char * 128).from_buffer_copy(id_bytes)
        check(lib().rb_comm_init_rank(ctx._h, n_ranks, rank, buf, C.byref(self._h)), "rb_comm_init_rank")

    @staticmethod
    def unique_id() -> bytes:
        buf = (C.c_char * 128)()
        check(lib().rb_comm_unique_id(buf), "rb_comm_unique_id")
        return bytes(buf)

    @classmethod
    def all(cls, ctxs: Sequence[Context]) -> "Comm":
        self = cls.__new__(cls)
        self._h, self._ctxs = C.c_void_p(), list(ctxs)
        arr = (C.c_void_p * len(ctxs))(*[c._h for c in ctxs])
        check(lib().rb_comm_init_all(arr, len(ctxs), C.byref(self._h)), "rb_comm_init_all")
        return self

    @property
    def transport(self) -> str:
        """"p2p ..." (k_mix_exchange over NVLink peer memory) or "nccl ... (why)" -- known after the first render_mix_allreduce."""
        buf = C.create_string_buffer(400)
        check(lib().rb_comm_transport(self._h, buf, 400), "rb_comm_transport")
        return buf.value.decode()

    def render_mix_allreduce(self, batches):
        """Render the batch of every local rank and sum the mixes over all ranks in place (asynchronous like a render)."""
        batches = [batches] if isinstance(batches, Batch) else list(batches)
        arr = (C.c_void_p * len(batches))(*[b._h for b in batches])
        check(lib().rb_batch_render_mix_allreduce(arr, len(batches), self._h), "rb_batch_render_mix_allreduce")

    def close(self):
        if self._h:
            lib().rb_comm_destroy(self._h)
            self._h = C.c_void_p()


_default_ctx: dict = {}


def default_context(device: int = 0) -> Context:
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


def flatten_sources(sources: Sequence[Source]) -> List[Source]:
    """`sources` followed by every second input of a mix() inside them (depth first): the descriptor array of a batch."""
    flat = list(sources)
    i = 0
    while i < len(flat):
        for e in flat[i].effects:
            if e.kind in (capi.RB_FX_MIX, capi.RB_FX_APPEND) and e.other is not None and not any(e.other is f for f in flat):
                flat.append(e.other)
        i += 1
    return flat


def pack_descs(sources: Sequence[Source], mix_starts: Optional[Sequence[int]] = None):
    """Build the rb_stream_desc array for `sources` (returns the array and the objects it points into).  Second inputs of a
    mix() are appended as descriptors of their own with mix_start = RB_MIX_START_CONSUMED."""
    flat = flatten_sources(sources)
    n = len(flat)
    descs = (capi.rb_stream_desc * max(1, n))()
    keep = [flat]
    for i, s in enumerate(flat):
        fx = (capi.rb_effect * max(1, len(s.effects)))()
        for j, e in enumerate(s.effects):
            fx[j].kind = e.kind
            for k in range(3):
                fx[j].u32[k] = e.u32[k]
            for k in range(12):
                fx[j].f32[k] = e.f32[k]
            for k in range(2):
                fx[j].ns[k] = e.ns[k]
            if e.kind in (capi.RB_FX_MIX, capi.RB_FX_APPEND) and e.other is not None:
                fx[j].u32[0] = next(k for k, f in enumerate(flat) if f is e.other)
        keep.append(fx)
        d = descs[i]
        d.sample_rate = s.base_rate
        d.channels = s.base_channels
        d.format = s.fmt_override if s.fmt_override is not None else _FMT_OF_NP[s.pcm.dtype]
        d.n_samples = s.pcm.size
        d.span_len = s.span_len
        d.n_effects = len(s.effects)
        d.effects = C.cast(fx, C.POINTER(capi.rb_effect))
        if i >= len(sources):
            d.mix_start = capi.RB_MIX_START_CONSUMED
        else:
            d.mix_start = int(mix_starts[i]) if mix_starts is not None else 0
    return descs, keep


def plan(source: Source, mixer_channels: int, mixer_rate: int):
    """Host-only closed forms for one source: (samples the mixer pulls, chain channels, chain rate, chain samples)."""
    descs, keep = pack_descs([source])
    n, ch, rate, cn = C.c_uint64(), C.c_uint16(), C.c_uint32(), C.c_uint64()
    if len(keep[0]) > 1:      # the source names others (mix, from_iter): plan it inside its descriptor array
        check(lib().rb_streams_plan(descs, len(keep[0]), 0, mixer_channels, mixer_rate, C.byref(n), C.byref(ch), C.byref(rate),
                                    C.byref(cn)), "rb_streams_plan")
    else:
        check(lib().rb_stream_plan(C.byref(descs[0]), mixer_channels, mixer_rate, C.byref(n), C.byref(ch), C.byref(rate),
                                   C.byref(cn)), "rb_stream_plan")
    return n.value, ch.value, rate.value, cn.value


class Batch:
    """mixer(channels, rate) + Mixer::add for every source, as one rb_batch."""

    def __init__(self, sources: Sequence[Source], mixer_channels: int, mixer_rate: int, flags: int = 0,
                 mix_starts: Optional[Sequence[int]] = None, ctx: Optional[Context] = None, master: Sequence[Effect] = ()):
        """master: adapters on the MixerSource itself, [amplify] [limit] [amplify] (rb_batch_set_master)."""
        self.ctx = ctx or default_context()
        self._descs, self._keep = pack_descs(list(sources), mix_starts)
        self.sources = self._keep[0]          # the sources handed in, then the second inputs of their mix() adapters
        self._h = C.c_void_p()
        check(lib().rb_batch_create(self.ctx._h, mixer_channels, mixer_rate, self._descs, len(self.sources), flags,
                                    C.byref(self._h)), "rb_batch_create")
        if master:
            try:
                check(lib().rb_batch_set_master(self._h, effect_records(master), len(master)), "rb_batch_set_master")
            except Exception:
                self.close()
                raise

    def close(self):
        if self._h:
            lib().rb_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def upload(self, i: int, pcm: Optional[np.ndarray] = None):
        a = self.sources[i].pcm if pcm is None else np.ascontiguousarray(pcm)
        check(lib().rb_batch_upload(self._h, i, a.ctypes.data_as(C.c_void_p), a.size), "rb_batch_upload")

    def upload_all(self):
        for i in range(len(self.sources)):
            self.upload(i)

    def upload_packed(self, host_ptr: int, total_samples: int):
        check(lib().rb_batch_upload_packed(self._h, C.c_void_p(host_ptr), total_samples), "rb_batch_upload_packed")

    def input_device_ptr(self, i: int) -> Tuple[int, int]:
        p, cap = C.c_void_p(), C.c_uint64()
        check(lib().rb_batch_input_device_ptr(self._h, i, C.byref(p), C.byref(cap)), "rb_batch_input_device_ptr")
        return p.value or 0, cap.value

    def stream_out_len(self, i: int) -> int:
        n = C.c_uint64()
        check(lib().rb_batch_stream_out_len(self._h, i, C.byref(n)), "rb_batch_stream_out_len")
        return n.value

    @property
    def mix_len(self) -> int:
        n = C.c_uint64()
        check(lib().rb_batch_mix_len(self._h, C.byref(n)), "rb_batch_mix_len")
        return n.value

    @property
    def launches_per_render(self) -> int:
        n = C.c_uint32()
        check(lib().rb_batch_launches_per_render(self._h, C.byref(n)), "rb_batch_launches_per_render")
        return n.value

    @property
    def kernel_family(self) -> int:
        """-1 general path, 0 k_fused_biquad / k_fused_nobiquad, 1 k_fused_hot, 2 k_fused_lanes."""
        n = C.c_int()
        check(lib().rb_batch_kernel_family(self._h, C.byref(n)), "rb_batch_kernel_family")
        return n.value

    @property
    def mix_group(self) -> int:
        """Streams per partial sum of the fused mixer sum (0: one sequential sum), see rb_batch_mix_group."""
        n = C.c_uint32()
        check(lib().rb_batch_mix_group(self._h, C.byref(n)), "rb_batch_mix_group")
        return n.value

    @property
    def algorithmic_bytes(self) -> int:
        n = C.c_uint64()
        check(lib().rb_batch_algorithmic_bytes(self._h, C.byref(n)), "rb_batch_algorithmic_bytes")
        return n.value

    def render_mix_device(self):
        check(lib().rb_batch_render_mix_device(self._h), "rb_batch_render_mix_device")

    @property
    def mix_device_ptr(self) -> int:
        p = C.c_void_p()
        check(lib().rb_batch_mix_device_ptr(self._h, C.byref(p)), "rb_batch_mix_device_ptr")
        return p.value or 0

    def render_mix(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        n = self.mix_len
        if out is None:
            out = np.empty(n, dtype=np.float32)
        w = C.c_uint64()
        check(lib().rb_batch_render_mix(self._h, out.ctypes.data_as(C.c_void_p), out.size, C.byref(w)),
              "rb_batch_render_mix")
        return out[: w.value]

    def render_mix_into(self, host_ptr: int, max_samples: int) -> int:
        w = C.c_uint64()
        check(lib().rb_batch_render_mix(self._h, C.c_void_p(host_ptr), max_samples, C.byref(w)), "rb_batch_render_mix")
        return w.value

    def read_mix(self, offset: int, n: int) -> np.ndarray:
        """A block of the rendered mixer output (what a block-pulling `Source` shim hands out)."""
        out = np.empty(n, dtype=np.float32)
        w = C.c_uint64()
        check(lib().rb_batch_read_mix(self._h, offset, out.ctypes.data_as(C.c_void_p), n, C.byref(w)), "rb_batch_read_mix")
        return out[: w.value]

    def read_stream(self, i: int) -> np.ndarray:
        n = self.stream_out_len(i)
        out = np.empty(n, dtype=np.float32)
        w = C.c_uint64()
        check(lib().rb_batch_read_stream(self._h, i, out.ctypes.data_as(C.c_void_p), n, C.byref(w)),
              "rb_batch_read_stream")
        return out[: w.value]


# ---------------------------------------------------------------------------------------------
# mixer::mixer(channels, sample_rate) -> (Mixer, MixerSource)   src/mixer.rs:25-43
# ---------------------------------------------------------------------------------------------
class Session:
    """Streaming mixer: sources whose PCM arrives block by block (decoders, live input), the mixer output pulled block by
    block -- the block form of MixerSource::next (src/mixer.rs:120-136).  Any split into pushes and renders gives the
    bytes of the whole-stream Batch render with RB_FUSED_LANES.  `sources` describe the chains
    (UniformSourceIterator(src, 1, rate)[.low_pass / .high_pass][.amplify]); their pcm is ignored.  A chain may begin with a push
    program -- fade_in / fade_out / linear_gain_ramp / take_duration / distortion, with amplify and speed among them -- applied as
    the PCM is pushed; a take ends its source, and later pushes are dropped (include/rodio_b200.h has the takes served)."""

    def __init__(self, sources: Sequence[Source], mixer_rate: int, fifo_frames: int = 8192, max_block_frames: int = 4096,
                 mix_starts: Optional[Sequence[int]] = None, ctx: Optional[Context] = None, mixer_channels: Optional[int] = None,
                 master: Sequence[Effect] = (), restarts: bool = False):
        """master: adapters on the mixer's output, [amplify] [limit] [amplify] (rb_session_set_master).
        restarts: RB_SESSION_RESTARTS -- the mixer's conversion restarts where rodio's does: every min(span_len, 32768) samples of
        a source that reports a span (a SamplesBuffer reports its length), and behind take_duration (include/rodio_b200.h)."""
        self.ctx = ctx or default_context()
        self.sources = list(sources)
        self.max_block_frames = max_block_frames
        # mixer(channels, rate): the chains end in UniformSourceIterator(_, channels, rate), so they report the mixer's count
        self.channels = mixer_channels or (self.sources[0].channels() if self.sources else 1)
        self.src_channels = [s.base_channels for s in self.sources]       # what is pushed: the source's own interleaving
        # generator sources (RB_FX_SIGNAL) fill themselves and take no pushes: the push helpers pass them by
        self.generators = [bool(s.effects) and s.effects[0].kind == capi.RB_FX_SIGNAL for s in self.sources]
        self._descs, self._keep = pack_descs(self.sources, mix_starts)
        self._h = C.c_void_p()
        if restarts:
            check(lib().rb_session_create_ex(self.ctx._h, self.channels, mixer_rate, self._descs, len(self.sources), fifo_frames,
                                             max_block_frames, capi.RB_SESSION_RESTARTS, C.byref(self._h)), "rb_session_create_ex")
        else:
            check(lib().rb_session_create(self.ctx._h, self.channels, mixer_rate, self._descs, len(self.sources), fifo_frames,
                                          max_block_frames, C.byref(self._h)), "rb_session_create")
        if master:
            try:
                self.set_master(master)
            except Exception:
                self.close()
                raise

    def set_master(self, effects: Sequence[Effect]):
        """mixer_source.amplify(a).limit(s).amplify(b) on the output; before the first rendered frame."""
        check(lib().rb_session_set_master(self._h, effect_records(effects), len(effects)), "rb_session_set_master")

    def close(self):
        if self._h:
            lib().rb_session_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def push(self, stream: int, pcm, end_of_stream: bool = False, spans: Optional[Sequence[Tuple[int, int]]] = None):
        """spans: [(at, span_len), ...] -- after `at` samples of this push the source's current_span_len() is span_len (0: None),
        for a session with restarts (rb_session_push_spans); None or empty: the report stays as it is."""
        a = np.ascontiguousarray(pcm, dtype=np.float32)
        ch = self.src_channels[stream]
        assert a.size % ch == 0, "whole frames"
        if spans:
            m = _span_marks(spans)
            check(lib().rb_session_push_spans(self._h, stream, a.ctypes.data_as(C.c_void_p), a.size // ch, m, len(spans), int(end_of_stream)),
                  "rb_session_push_spans")
            return
        check(lib().rb_session_push(self._h, stream, a.ctypes.data_as(C.c_void_p), a.size // ch, int(end_of_stream)), "rb_session_push")

    def push_packed(self, blocks: Sequence[np.ndarray], end_of_stream: Optional[Sequence[bool]] = None,
                    spans: Optional[Sequence[Sequence[Tuple[int, int]]]] = None):
        """One block per source (possibly empty), pushed with one copy and one kernel.  spans: one list of (at, span_len) marks per
        source, as in push (rb_session_push_packed_spans).  The entries of generator sources are passed by."""
        assert len(blocks) == len(self.sources)
        blocks = [np.zeros(0, np.float32) if g else np.ascontiguousarray(b, dtype=np.float32) for b, g in zip(blocks, self.generators)]
        if end_of_stream is not None:
            end_of_stream = [bool(e) and not g for e, g in zip(end_of_stream, self.generators)]
        if spans is not None:
            spans = [() if g else sp for sp, g in zip(spans, self.generators)]
        flat = np.concatenate(blocks) if blocks else np.zeros(0, np.float32)
        n = (C.c_uint64 * len(blocks))(*[b.size // ch for b, ch in zip(blocks, self.src_channels)])
        eos = (C.c_uint8 * len(blocks))(*[int(bool(e)) for e in end_of_stream]) if end_of_stream is not None else None
        if spans is not None:
            assert len(spans) == len(self.sources)
            counts = (C.c_uint32 * len(blocks))(*[len(m) for m in spans])
            m = _span_marks([x for sp in spans for x in sp])
            check(lib().rb_session_push_packed_spans(self._h, flat.ctypes.data_as(C.c_void_p), n, eos, counts, m), "rb_session_push_packed_spans")
            return
        check(lib().rb_session_push_packed(self._h, flat.ctypes.data_as(C.c_void_p), n, eos), "rb_session_push_packed")

    def push_silence(self, stream: int, n_frames: int):
        """Player::pause for `n_frames` frames: whole frames of 0.0 behind the source's push program, which is not pulled meanwhile
        (its fades and takes stand still), as Pausable does (src/source/pausable.rs:85-97).  Refused for a filter in front."""
        check(lib().rb_session_push_silence(self._h, stream, int(n_frames)), "rb_session_push_silence")

    def start(self, stream: int):
        """Mixer::add for a source created with mix_start = capi.RB_SESSION_HELD: joins at the frame rendered next."""
        check(lib().rb_session_start(self._h, stream), "rb_session_start")

    def follow(self, stream: int, predecessor: int):
        """Queue a held source behind another one (Player::append): it starts on the frame after that one has played out."""
        check(lib().rb_session_follow(self._h, stream, predecessor), "rb_session_follow")

    def skip(self, stream: int):
        """Player::skip_one / stop for this source: it ends with the last frame the converter has pulled (rb_session_skip)."""
        check(lib().rb_session_skip(self._h, stream), "rb_session_skip")

    def set_amplify(self, stream: int, factor: float):
        """Amplify::set_factor on the chain's AMPLIFY of a live source: applies from the next rendered block on."""
        check(lib().rb_session_set_amplify(self._h, stream, float(factor)), "rb_session_set_amplify")

    def set_volume(self, stream: int, factor: float):
        """Player::set_volume (src/player.rs:180-186): the AMPLIFY in FRONT of the mixer's conversion (behind a filter in front
        of it, where the Player keeps its own, src/player.rs:120-128), for every frame the converter pulls from now on."""
        check(lib().rb_session_set_volume(self._h, stream, float(factor)), "rb_session_set_volume")

    def source_runs(self, stream: int) -> int:
        """Converter runs of the source that have produced an output so far (rb_session_source_runs)."""
        n = C.c_uint64()
        check(lib().rb_session_source_runs(self._h, stream, C.byref(n)), "rb_session_source_runs")
        return n.value

    def restart_launches(self) -> int:
        """Launches of the lane kernel's RESTART variants so far: only blocks in which a source restarts make one."""
        n = C.c_uint64()
        check(lib().rb_session_restart_launches(self._h, C.byref(n)), "rb_session_restart_launches")
        return n.value

    def available(self) -> Tuple[int, bool]:
        n, e = C.c_uint64(), C.c_int()
        check(lib().rb_session_available(self._h, C.byref(n), C.byref(e)), "rb_session_available")
        return n.value, bool(e.value)

    def render(self, max_frames: Optional[int] = None) -> Tuple[np.ndarray, bool]:
        """Up to max_frames mixer frames; (interleaved samples, ended) -- ended: MixerSource::next() would return None from
        here on."""
        cap = self.max_block_frames if max_frames is None else min(int(max_frames), self.max_block_frames)
        out = np.empty(cap * self.channels, dtype=np.float32)
        n, e = C.c_uint64(), C.c_int()
        check(lib().rb_session_render(self._h, out.ctypes.data_as(C.c_void_p), cap, C.byref(n), C.byref(e)), "rb_session_render")
        return out[: n.value * self.channels].copy(), bool(e.value)

    def get_state(self) -> bytes:
        n = C.c_uint64()
        check(lib().rb_session_get_state(self._h, None, 0, C.byref(n)), "rb_session_get_state")
        buf = (C.c_uint8 * n.value)()
        check(lib().rb_session_get_state(self._h, buf, n.value, C.byref(n)), "rb_session_get_state")
        return bytes(buf)

    def set_state(self, blob: bytes):
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        check(lib().rb_session_set_state(self._h, buf, len(blob)), "rb_session_set_state")


def _span_marks(spans):
    """rb_span_mark array of [(at, span_len), ...] (None when empty)."""
    if not spans:
        return None
    return (capi.rb_span_mark * len(spans))(*[capi.rb_span_mark(int(at), int(span), 0) for at, span in spans])


class _MixerShared:
    def __init__(self, channels, rate, flags, ctx):
        self.channels, self.rate, self.flags, self.ctx = channels, rate, flags, ctx
        self.sources: List[Source] = []
        self.starts: List[int] = []
        self.pos = 0              # samples already handed out by MixerSource
        self.rendered: Optional[np.ndarray] = None
        self.active: Optional[np.ndarray] = None
        self.rendered_master: Tuple[Effect, ...] = ()   # the MixerSource adapters `rendered` went through


class Mixer:
    """The input handle (`mixer::Mixer`, src/mixer.rs:47-66). `add` is infallible like the reference."""

    def __init__(self, shared: _MixerShared):
        self._s = shared

    def add(self, source: Source):
        s = self._s
        s.sources.append(source)
        s.starts.append(s.pos)    # joins at the next frame boundary (mixer.rs:175-183), done by the library
        s.rendered = None


class MixerSource:
    """The output (`mixer::MixerSource`, src/mixer.rs:70-136): an iterator of f32 that implements Source."""

    def __init__(self, shared: _MixerShared, master: Tuple[Effect, ...] = ()):
        self._s = shared
        self._master = tuple(master)

    # -- adapters on the MixerSource itself: [amplify] [limit] [amplify] (rb_batch_set_master), over the whole mix ----------
    def amplify(self, value: float) -> "MixerSource":
        """Source::amplify on the mixer's output (src/source/amplify.rs:63-65).  A new handle on the same mixer: rodio's
        adapters take the source by value."""
        return MixerSource(self._s, self._master + (amplify_effect(value),))

    def limit(self, settings: Optional[LimitSettings] = None) -> "MixerSource":
        """Source::limit on the mixer's output (src/source/limit.rs:94-130), built for the mixer's channels and rate."""
        return MixerSource(self._s, self._master + (limit_effect(settings),))

    def channels(self) -> int:
        return self._s.channels

    def sample_rate(self) -> int:
        return self._s.rate

    def current_span_len(self):
        return None

    def try_seek(self, pos):
        raise capi.RodioB200Error(capi.RB_ERR_NOT_SUPPORTED_SEEK, "MixerSource::try_seek",
                                  "SeekError::NotSupported (src/mixer.rs:109-113)")

    def _render(self):
        s = self._s
        if s.rendered is not None and s.rendered_master == self._master:
            return
        s.rendered_master = self._master
        if not s.sources:
            s.rendered = np.zeros(0, dtype=np.float32)
            s.active = np.zeros(0, dtype=bool)
            return
        with Batch(s.sources, s.channels, s.rate, flags=s.flags, mix_starts=s.starts, ctx=s.ctx, master=self._master) as b:
            b.upload_all()
            s.rendered = b.render_mix()
            act = np.zeros(s.rendered.size + 1, dtype=np.int64)
            for i in range(len(s.sources)):
                n = b.stream_out_len(i)
                if n:
                    st = (s.starts[i] + s.channels - 1) // s.channels * s.channels
                    act[st] += 1
                    act[st + n] -= 1
            s.active = np.cumsum(act)[:-1] > 0

    def next(self) -> Optional[float]:
        """Iterator::next — None when no source is playing at this position (src/mixer.rs:131-135)."""
        s = self._s
        self._render()
        p = s.pos
        s.pos += 1
        if p < s.rendered.size and s.active[p]:
            return float(s.rendered[p])
        return None

    def __iter__(self):
        return self

    def __next__(self):
        v = self.next()
        if v is None:
            raise StopIteration
        return v

    def collect(self) -> np.ndarray:
        """Drain until the mixer first reports None."""
        s = self._s
        self._render()
        p = s.pos
        q = p
        while q < s.rendered.size and s.active[q]:
            q += 1
        s.pos = q + 1
        return s.rendered[p:q].copy()


def mixer(channels: int, sample_rate: int, flags: int = 0, ctx: Optional[Context] = None) -> Tuple[Mixer, MixerSource]:
    """mixer::mixer(channels, sample_rate) — src/mixer.rs:25-43."""
    if channels <= 0 or sample_rate <= 0:
        raise ValueError("channels and sample_rate must be non-zero")
    sh = _MixerShared(int(channels), int(sample_rate), flags, ctx)
    return Mixer(sh), MixerSource(sh)


# ---------------------------------------------------------------------------------------------
# Player ("Sink" in rodio <= 0.20): the control handle, on blocks        src/player.rs:20-351
# ---------------------------------------------------------------------------------------------
class Player:
    """`Player::connect_new(&mixer)` + `append` / `set_volume` / `set_speed` / `len` / `empty` for offline drains.

    rodio wraps every appended source in speed -> track_position -> pausable -> amplify(volume) -> skippable ->
    stoppable (src/player.rs:122-166) and samples the controls every 5 ms of audio.  On blocks the controls are
    read when a source is appended: its chain becomes `source.speed(speed).amplify(volume)` and it is queued
    behind the sources appended before it (src/queue.rs: one source after the other, each converted to the
    mixer's format on its own); `pause()` / `play()` at known positions are the `pauses` of `append` (Pausable sits between the
    speed and the volume, player.rs:122-128: the source and its filters are not pulled while paused, whole frames of zeros go
    out -- RB_FX_PAUSE).  This class renders offline; the controls WHILE playing live on a `Session`: `follow` (append),
    `set_volume` (the Amplify in front of the mixer's conversion, per pulled frame), pausing = `push_silence` (frames of zeros
    behind the source's fades and takes, which stand still), stop / skip = end_of_stream (INTEGRATION.md, examples/live_player.c).  Seeking is a control-plane feature of the decoders and out of
    scope (SURVEY.md §2)."""

    def __init__(self, mixer: "Mixer"):
        self._mixer = mixer
        self._volume = 1.0
        self._speed = 1.0
        self._next_start = mixer._s.pos
        self._count = 0

    @staticmethod
    def connect_new(mixer: "Mixer") -> "Player":
        return Player(mixer)

    def volume(self) -> float:
        return self._volume

    def set_volume(self, value: float):
        """Player::set_volume — multiplies every sample (src/player.rs:180-186); == Source::amplify(value)."""
        self._volume = float(value)

    def speed(self) -> float:
        return self._speed

    def set_speed(self, value: float):
        """Player::set_speed (src/player.rs:203-207): rescales the reported sample rate like Source::speed."""
        self._speed = float(value)

    def append(self, source: Source, pauses: Sequence[Tuple[int, int]] = ()):
        """Player::append — src/player.rs:104-170.  `pauses`: (sample of the source at which Player::pause() is observed, frames of
        silence until Player::play()), in increasing order of the sample -- positions count the source's own samples."""
        s = self._mixer._s
        chain = source.speed(self._speed)
        shift = 0
        for at, frames in pauses:                       # a later pause sees the zeros of the earlier ones in front of it
            chain = chain.pause_at(int(at) + shift, int(frames))
            shift += int(frames) * chain.channels()
        chain = chain.amplify(self._volume)
        n = plan(chain, s.channels, s.rate)[0]
        start = (self._next_start + s.channels - 1) // s.channels * s.channels
        s.sources.append(chain)
        s.starts.append(start)
        s.rendered = None
        self._next_start = start + n
        self._count += 1

    def len(self) -> int:
        return self._count

    def empty(self) -> bool:
        return self._count == 0


# ---------------------------------------------------------------------------------------------
# conversions::{SampleRateConverter, ChannelCountConverter, SampleTypeConverter}
# ---------------------------------------------------------------------------------------------
def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).reshape(-1)


def SampleRateConverter(input, from_rate: int, to_rate: int, num_channels: int, ctx: Optional[Context] = None) -> np.ndarray:
    """conversions::SampleRateConverter::new(input, from, to, channels).collect() — sample_rate.rs:52-201."""
    x = _f32(input)
    ctx = ctx or default_context()
    n = C.c_uint64()
    check(lib().rb_sample_rate_out_len(x.size, from_rate, to_rate, num_channels, C.byref(n)), "rb_sample_rate_out_len")
    out = np.empty(n.value, dtype=np.float32)
    check(lib().rb_convert_sample_rate(ctx._h, x.ctypes.data_as(C.c_void_p), x.size, from_rate, to_rate, num_channels,
                                       out.ctypes.data_as(C.c_void_p), out.size, C.byref(n)), "rb_convert_sample_rate")
    return out[: n.value]


def ChannelCountConverter(input, from_channels: int, to_channels: int, ctx: Optional[Context] = None) -> np.ndarray:
    """conversions::ChannelCountConverter::new(input, from, to).collect() — channels.rs:28,:57-85."""
    x = _f32(input)
    ctx = ctx or default_context()
    n = C.c_uint64()
    check(lib().rb_channels_out_len(x.size, from_channels, to_channels, C.byref(n)), "rb_channels_out_len")
    out = np.empty(n.value, dtype=np.float32)
    check(lib().rb_convert_channels(ctx._h, x.ctypes.data_as(C.c_void_p), x.size, from_channels, to_channels,
                                    out.ctypes.data_as(C.c_void_p), out.size, C.byref(n)), "rb_convert_channels")
    return out[: n.value]


def SampleTypeConverter(input: np.ndarray, out_fmt: int, in_fmt: Optional[int] = None, ctx: Optional[Context] = None) -> np.ndarray:
    """conversions::SampleTypeConverter::<_, O>::new(input).collect() — sample.rs:14,:42-44."""
    x = np.ascontiguousarray(input).reshape(-1)
    if in_fmt is None:
        in_fmt = _FMT_OF_NP[x.dtype]
    ctx = ctx or default_context()
    odt = np.int32 if out_fmt == capi.RB_FMT_I24_IN_I32 else _NP_OF_FMT[out_fmt]
    out = np.empty(x.size, dtype=odt)
    check(lib().rb_convert_samples(ctx._h, x.ctypes.data_as(C.c_void_p), in_fmt, out.ctypes.data_as(C.c_void_p),
                                   out_fmt, x.size), "rb_convert_samples")
    return out
