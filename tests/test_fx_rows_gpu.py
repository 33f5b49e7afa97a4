"""k_fused_fx on batches whose streams differ: lengths around a tile, a group of four and the RMS window, echo delays around the
input length and around the edge of the interior front path, late joiners, every front and back shape the planner takes, per-row
AGC and limiter settings, AGC input that drives the running sum through its residue and through inf / NaN, and an exact-order
chain of more than two waves of CTAs.

k_fused_fx (rb_fx.cu) runs a 7-slot tile pipeline: the workers compute the front of tile `it`, chains P and S walk `it - 1`, the
desired gain is `it - 2`, chain G `it - 3` and the output `it - 4` (with a limiter: chain L `it - 5`, the output `it - 6`).  Every
chain walks ceil(n / 4) groups of four samples of a tile, the tail group padded with zeros, and a CTA walks the tiles of its
longest stream.  The designs below put those edges where they can be seen: a stream that borrows another stream's tile count,
drops its tail group, takes the echo tap one sample early or writes its partial row at the wrong mix start changes the output.

Every design is checked three ways:
  * bit for bit: the default launch against the oracle's per-stream outputs added in the kernel's documented order (the four
    streams of a CTA from +0.0 at their mix start, then the partial rows in CTA order), and within 1e-5 * peak of the oracle's
    sequential mixer; the exact-order chain against the sequential mixer itself.  NaNs compare as NaNs: the NaN masks must be
    identical, the payloads are not compared (the host and the device produce different ones);
  * against a float64 restatement written here with numpy from the reference sources (channel_volume.rs, spatial.rs, delay.rs +
    mix.rs, agc.rs with its RMS window summed from the ring itself, limit.rs), with Rust's rules for non-finite values
    (f32::min / max ignore NaN, clamp passes NaN through, a comparison with NaN is false).  It shares no code with the oracle;
  * on the CPU, the oracle against the f64 restatement on every design (lengths, NaN masks, a stated distance bound), so that a
    misreading of agc.rs or limit.rs that the kernel and the oracle share would show."""
import functools
import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import pytest

import oracle
import rodio_b200 as rb
from helpers import noise, to_oracle
from rodio_b200 import capi

RATE = 48000
FX_R = 4                        # streams per CTA (rb_fx.cu)
TILE = 256                      # samples per stream and tile
RMS_WINDOW = 8192               # agc.rs RMS_WINDOW_SIZE
H100_SMS = 132                  # the SM count the CPU tests design for
LEFT, RIGHT = (-1.0, 0.0, 0.0), (1.0, 0.0, 0.0)
MIN_POSITIVE = float(np.finfo(np.float32).tiny)      # f32::MIN_POSITIVE (limit.rs:862)
# f64 bar on the device: the kernel may be at most this many times further from the f64 mix than the oracle's own mix, plus
# 1e-7 * peak (the rule of test_hot_rows_gpu.py).  The default launch adds the same per-stream samples in another order (per CTA,
# then the partial rows), which test_f64_restatement_matches_oracle keeps within 1.5x of the oracle's distance.
F64_FACTOR = 2.0


def stream_tol(n):
    """Bound between the oracle (f32) and the f64 restatement over n samples, relative to the peak.  The AGC's gain recurrence
    g * k + d * (1 - k) has k within 5e-6 of 1 (attack times of seconds), so it keeps each rounding of g for some 100 000
    samples: over n samples its three roundings per sample (two products, one sum, each at most 2^-24 relative) can add up to
    3 n 2^-24 if they go the same way.  The running f32 sum of squares behind rms_gain drifts at the same rate; the other
    roundings (sqrt, the divisions, the limiter's log2 / exp2) are single ones.  Streams of up to 1000 samples get the bound of
    1000.  The worst stream here (agc_limit_mono: 9 017 samples, 10 s attack and release) stays 3.6x inside its bound; a misread branch or
    coefficient is off by percents."""
    return 3.0 * max(n, 1000) * 2.0 ** -24


def ns_for(delay, ch):
    """The shortest Duration (ns) whose reverb delays by `delay` samples of a `ch`-channel 48 kHz stream (delay.rs:8-16)."""
    ns = -(-delay * 1_000_000_000 // (ch * RATE))
    assert delay_samples(ns, ch) == delay
    return ns


def delay_samples(ns, ch):
    return ns * ch * RATE // 1_000_000_000


@dataclass
class Row:
    pcm: np.ndarray                              # f32, interleaved, the mixer's channel count
    start: int = 0                               # mix start, samples
    cv: Optional[Tuple[str, tuple]] = None       # ("spatial", emitter) or ("volume", volumes)
    delay: Optional[int] = None                  # reverb delay in samples (the Duration is ns_for(delay))
    amp: float = 0.4                             # reverb amplitude
    agc: Optional[rb.AutomaticGainControlSettings] = None
    lim: Optional[rb.LimitSettings] = None
    # (sample, reason): from this sample of the stream on, f32 and f64 legitimately take different branches; the f64 comparison
    # stops there (lengths and NaN masks are still compared over the whole stream)
    branch: Optional[Tuple[int, str]] = None


@dataclass
class Case:
    name: str
    ch: int
    rows: List[Row]
    launches: Tuple[str, ...] = ("default", "chain")
    family: int = 5                              # the kernel family of the default launch (-1: the general path)

    @property
    def starts(self):
        return [r.start for r in self.rows]

    def sources(self):
        out = []
        for r in self.rows:
            s = rb.TestSource(r.pcm, self.ch, RATE)
            if r.cv is not None:
                kind, p = r.cv
                s = rb.Spatial(s, list(p), list(LEFT), list(RIGHT)) if kind == "spatial" else rb.ChannelVolume(s, list(p))
            if r.delay is not None:
                s = s.reverb(rb.Duration.from_nanos(ns_for(r.delay, self.ch)), r.amp)
            if r.agc is not None:
                s = s.automatic_gain_control(r.agc)
            if r.lim is not None:
                s = s.limit(r.lim)
            out.append(s)
        return out

    def out_len(self, r):
        return r.pcm.size + (r.delay or 0)


# ------------------------------------------------------------------ the float64 restatement
def coefficient(ns):
    """math.rs duration_to_coefficient: exp(-1 / (Duration::as_secs_f32() * rate)), a zero duration gives exp(-inf) = 0.  The
    reference stores the coefficient as an f32 parameter, so the restatement takes it in f32 too (numpy's expf): near 1 the
    rounding of k is a relative error of up to 1 % in 1 - k, which would otherwise dominate every AGC comparison."""
    F = np.float32
    secs = F(ns // 1_000_000_000) + F(ns % 1_000_000_000) / F(1e9)
    with np.errstate(divide="ignore"):
        return float(np.exp(F(-1.0) / (secs * F(RATE))))


def spatial_volumes64(emitter):
    """spatial.rs:48-69 in f64 (the positions are the f32 values)."""
    f = lambda p: [float(np.float32(v)) for v in p]
    e, l, r = f(emitter), f(LEFT), f(RIGHT)
    d2 = lambda a, b: sum((x - y) ** 2 for x, y in zip(a, b))
    ld2, rd2 = d2(l, e), d2(r, e)
    md = math.sqrt(d2(l, r))
    ld, rd = math.sqrt(ld2), math.sqrt(rd2)
    lm = min(((ld - rd) / md + 1.0) / 4.0 + 0.5, 1.0)
    rm = min(((rd - ld) / md + 1.0) / 4.0 + 0.5, 1.0)
    return [lm * min(1.0 / ld2, 1.0), rm * min(1.0 / rd2, 1.0)]


def front64(r, ch):
    """channel_volume.rs:71-88 (every frame averaged to mono, times the channel's volume), then reverb = Mix(x, Delay(Amplify(x)))
    (source/mod.rs:628-634): x[n] + amp * x[n - D] while the input lasts, the delayed copy alone for D samples more."""
    x = r.pcm.astype(np.float64)
    if r.cv is not None:
        kind, p = r.cv
        vols = spatial_volumes64(p) if kind == "spatial" else [float(np.float32(v)) for v in p]
        mono = x.reshape(-1, ch).sum(axis=1) / ch
        x = (mono[:, None] * np.asarray(vols, dtype=np.float64)[None, :]).reshape(-1)
    if r.delay is not None:
        y = np.zeros(x.size + r.delay)
        y[:x.size] += x
        y[r.delay:] += float(np.float32(r.amp)) * x
        x = y
    return x


def window_sums(q):
    """The RMS window of agc.rs (CircularBuffer: the last 8192 squares, zeros before the first) summed from its contents for every
    sample: each window is a suffix of one block of 8192 plus a prefix of the next, both sums of non-negative terms, so nothing
    is ever subtracted and a window that holds only zeros sums to exactly 0."""
    R, T = q.shape
    W = RMS_WINDOW
    nb = -(-T // W) + 1
    p = np.zeros((R, nb * W))
    p[:, W:W + T] = q
    b = p.reshape(R, nb, W)
    with np.errstate(invalid="ignore"):
        pre = np.cumsum(b, axis=2)
        suf = np.cumsum(b[:, :, ::-1], axis=2)[:, :, ::-1]
        P = W + np.arange(T)
        k, o = P // W, P % W
        tail = np.where(o + 1 < W, suf[:, k - 1, np.minimum(o + 1, W - 1)], 0.0)
        return pre[:, k, o] + tail


def agc64(E, settings):
    """agc.rs:397-504 over the rows of E (interleaved samples, one state for all channels), the RMS from window_sums."""
    R, T = E.shape
    col = lambda f: np.asarray([f(s) for s in settings], dtype=np.float64)
    tg = col(lambda s: float(np.float32(s.target_level)))
    mg = col(lambda s: float(np.float32(s.absolute_max_gain)))
    fl = col(lambda s: float(np.float32(s.floor)))
    att = col(lambda s: coefficient(min(int(s.attack_time), 10_000_000_000)))      # source/mod.rs:432-433
    rel = col(lambda s: coefficient(min(int(s.release_time), 10_000_000_000)))
    V = np.abs(E)
    G = np.empty((R, T))
    with np.errstate(all="ignore"):
        rms = np.sqrt(window_sums(V * V) / RMS_WINDOW)
        rms_gain = np.where(rms > 0.0, tg[:, None] / rms, mg[:, None])
        peak, gain = np.zeros(R), np.ones(R)
        for n in range(T):
            v = V[:, n]
            c = np.where(v > peak, 0.0, rel)
            peak = peak * c + v * (1.0 - c)
            peak_gain = np.where(peak > 0.0, np.fmin(tg / peak, mg), mg)
            desired = np.fmax(np.fmin(rms_gain[:, n], peak_gain), fl)
            k = np.where(desired > gain, att, rel)
            g = gain * k + desired * (1.0 - k)
            gain = np.where(g < 0.1, 0.1, np.where(g > mg, mg, g))      # f32::clamp(0.1, max): NaN passes through
            G[:, n] = gain
        return E * G


def limit64(Y, settings, ch):
    """limit.rs:854-988: soft-knee gain computer in dB, per channel integrator = max(dB, release-smoothed) and attack-smoothed
    peak, the channels coupled by max(peaks) after the current channel's update, output * 10^(-max_peak / 20)."""
    R, T = Y.shape
    col = lambda f: np.asarray([f(s) for s in settings], dtype=np.float64)[:, None]
    thr = col(lambda s: float(np.float32(s.threshold)))
    knee = col(lambda s: float(np.float32(s.knee_width)))
    att = col(lambda s: coefficient(int(s.attack)))[:, 0]
    rel = col(lambda s: coefficient(int(s.release)))[:, 0]
    with np.errstate(all="ignore"):
        bias = 20.0 * np.log10(np.abs(Y) + MIN_POSITIVE) - thr
        kb = 2.0 * bias
        db = np.where(kb < -knee, 0.0, np.where(np.abs(kb) <= knee, (kb + knee) ** 2 / (8.0 * knee), bias))
        integ, pk = np.zeros((ch, R)), np.zeros((ch, R))
        M = np.empty((R, T))
        for n in range(T):
            c = n % ch
            integ[c] = np.fmax(db[:, n], rel * integ[c] + (1.0 - rel) * db[:, n])      # Float::max ignores NaN
            pk[c] = att * pk[c] + (1.0 - att) * integ[c]
            M[:, n] = pk[0] if ch == 1 else np.fmax(pk[0], pk[1])
        return Y * 10.0 ** (-M / 20.0)


def f64_streams(case):
    """Every stream of the case in f64; the AGC and the limiter walk the rows together (zero padding past a row's end does not
    reach its samples)."""
    xs = [front64(r, case.ch) for r in case.rows]
    T = max([x.size for x in xs] + [1])
    E = np.zeros((len(xs), T))
    for i, x in enumerate(xs):
        E[i, :x.size] = x
    if case.rows[0].agc is not None:
        E = agc64(E, [r.agc for r in case.rows])
    if case.rows[0].lim is not None:
        E = limit64(E, [r.lim for r in case.rows], case.ch)
    return [E[i, :x.size] for i, x in enumerate(xs)]


def f64_mix(case, ys):
    """The f64 streams summed at their mix starts, and the positions a comparison with it may use: those no stream reaches past
    its listed branch point."""
    n = max(r.start + y.size for r, y in zip(case.rows, ys))
    total, trust = np.zeros(n), np.ones(n, dtype=bool)
    for r, y in zip(case.rows, ys):
        total[r.start:r.start + y.size] += y
        if r.branch is not None:
            trust[r.start + r.branch[0]:r.start + y.size] = False
    return total, trust


# ------------------------------------------------------------------ the kernel's documented order and the comparisons
def insertion_order(starts):
    """The mixer's insertion order, in which a batch hands its streams to the kernels: by mix start, ties in array order
    (Mixer::add calls arrive in increasing output position, src/mixer.rs:175-183)."""
    return sorted(range(len(starts)), key=lambda i: starts[i])


def grouped_expected_mix(per_stream, starts, mix_len, group=FX_R):
    """k_fused_fx + k_fx_sum_partials: the streams in insertion order, per CTA of `group` streams added from +0.0 where each is
    active (at its mix start), then the partial rows added in CTA order starting from the first."""
    order = insertion_order(starts)
    per_stream, starts = [per_stream[i] for i in order], [starts[i] for i in order]
    total = None
    for g in range(0, len(per_stream), group):
        acc = np.zeros(mix_len, dtype=np.float32)
        for y, s in zip(per_stream[g:g + group], starts[g:g + group]):
            acc[s:s + y.size] = acc[s:s + y.size] + y
        total = acc if total is None else total + acc
    return total


def assert_same(got, want, what):
    """Bit for bit, except that NaNs compare as NaNs (identical masks, payloads not compared)."""
    assert got.shape == want.shape, f"{what}: length {got.shape} != {want.shape}"
    gn, wn = np.isnan(got), np.isnan(want)
    bad = np.nonzero(gn != wn)[0]
    assert bad.size == 0, f"{what}: NaN masks differ at {bad.size} samples, first at {bad[0]}: got {got[bad[0]]!r} want {want[bad[0]]!r}"
    g, w = got.view(np.uint32), want.view(np.uint32)
    bad = np.nonzero((g != w) & ~gn)[0]
    assert bad.size == 0, f"{what}: {bad.size}/{got.size} samples differ, first at {bad[0]}: got {got[bad[0]]!r} want {want[bad[0]]!r}"


def finite_distance(a, b, where=None):
    """max |a - b| and the peak of b over the positions where both are finite (and `where` holds)."""
    m = np.isfinite(a) & np.isfinite(b)
    if where is not None:
        m &= where
    if not m.any():
        return 0.0, 0.0
    a64, b64 = a[m].astype(np.float64), b[m].astype(np.float64)
    return float(np.max(np.abs(a64 - b64))), float(np.max(np.abs(b64)))


# ------------------------------------------------------------------ designed batches
AGC_DEFAULT = rb.AutomaticGainControlSettings()


def agc(target=1.0, attack_ms=4000, release_ms=0, max_gain=7.0, floor=0.0):
    return rb.AutomaticGainControlSettings(target_level=target, attack_time=rb.Duration.from_millis(attack_ms),
                                           release_time=rb.Duration.from_millis(release_ms), absolute_max_gain=max_gain, floor=floor)


AGC_ROWS = [    # per-row settings that reach the edges of the gain's range
    AGC_DEFAULT,
    agc(target=0.5, attack_ms=1, release_ms=0),                                 # the gain follows rms_gain sample by sample
    agc(target=0.8, attack_ms=30, release_ms=5, max_gain=5.0, floor=2.5),       # the floor lies above the settled gain
    agc(target=1.0, attack_ms=2, release_ms=2, max_gain=3.0),                   # quiet input: absolute_max_gain is reached
    agc(target=0.04, attack_ms=200, release_ms=1, max_gain=2.0),                # loud input: clamp(0.1, ...) holds the floor
    agc(target=0.6, attack_ms=20_000, release_ms=12_000, max_gain=4.0),         # times above 10 s are cut to 10 s
]
LIMITS = [rb.LimitSettings.default(), rb.LimitSettings.dynamic_content(), rb.LimitSettings.broadcast(), rb.LimitSettings.mastering(),
          rb.LimitSettings.live_performance(), rb.LimitSettings.gaming(), rb.LimitSettings.default().with_threshold(-9.0),
          rb.LimitSettings.default().with_threshold(-0.25).with_knee_width(1.0)]
AGC_AMP = (0.6, 0.6, 1.0, 0.01, 1.0, 0.3)     # input amplitude that takes AGC_ROWS[i] to its edge
# behind a burst: rms_gain = 0.2 / sqrt(residue / 8192) lies below max_gain for residues above 7 and below the peak gain of the
# quiet input, so the gain that follows the silence is the residue's (a negative one gives rms = NaN and max_gain)
AGC_BURST = agc(target=0.2, attack_ms=1, release_ms=0, max_gain=7.0)


def _sig(n, seed, amp=0.6):
    return noise(n, seed, amp)


def _stereo_lr(frames, seed, left, right):
    """Stereo noise whose channels differ in level, and swap levels halfway: the limiter's channel coupling is visible."""
    x = noise(2 * frames, seed).reshape(-1, 2)
    h = frames // 2
    x[:h, 0] *= left
    x[:h, 1] *= right
    x[h:, 0] *= right
    x[h:, 1] *= left
    return x.reshape(-1).astype(np.float32)


def _burst(seed, amp, burst, silence, quiet):
    """A loud burst, silence long enough for the burst to leave the RMS window, then quiet input: the f32 running sum keeps the
    residue of the burst, which may be positive, zero or negative."""
    return np.concatenate([noise(burst, seed, amp), np.zeros(silence, np.float32), noise(quiet, seed + 1, 0.01)]).astype(np.float32)


RESIDUE = "the burst has left the RMS window: f64 sums the ring to exactly 0, the f32 running sum keeps a residue whose sign picks rms_gain"
OVERFLOW = "squares of 1e20 overflow the f32 sum to inf and inf - inf = NaN once they leave the window; in f64 they do not overflow"
NAN_SUM = "a NaN square makes the f32 running sum NaN for the rest of the stream (rms_gain = max_gain); the f64 ring recovers after 8192 samples"
INF_SUM = "an infinite square leaves the f32 running sum NaN (inf - inf) once it leaves the window; the f64 ring sums to finite values again"


def _short_mono():
    """Streams shorter than a tile and than a group of four, lengths around a tile, one empty stream beside live ones; AGC with
    no front stage; the last CTA holds one stream."""
    lens = [0, 1, 3, 4, 5, 255, 256, 257, 1001]
    rows = [Row(_sig(L, 100 + i), agc=AGC_ROWS[i % 6]) for i, L in enumerate(lens)]
    return Case("short_mono_agc", 1, rows)


def _short_stereo():
    """Stereo Spatial -> reverb with odd delays -> AGC on frames 0, 1, 2, 127, 128, 129 (n_out odd, the tail group partial); the last
    CTA holds two streams."""
    frames = [0, 1, 2, 127, 128, 129, 1, 300, 64, 3]
    delays = [3, 5, 1, 999, 7, 255, 257, 1, 129, 11]
    rows = [Row(_sig(2 * f, 200 + i), cv=("spatial", (float(i % 5 - 2), 1.0, 0.5)), delay=d, agc=AGC_ROWS[i % 6])
            for i, (f, d) in enumerate(zip(frames, delays))]
    return Case("short_stereo_spatial_echo_agc", 2, rows)


def _window_mono():
    """Mono ChannelVolume -> reverb (336 samples) -> AGC: n_out just below and above 8192 (where the window starts dropping
    squares) and 8192 + delay (where the interior front path starts); a CTA whose streams end in different tiles, its longest one
    (several tiles longer) not first; a last CTA of three streams.  No mono length is a multiple of 4."""
    D = 336
    lens = [8191 - D, 8193 - D, 8191, 8193, 1003, 2999, 12001, 5, 8195, 8189, 9001]
    vols = [0.7, 1.3, -0.9, 0.5, 1.0, 0.25, 1.1, 2.0, 0.6, 0.8, 1.2]
    rows = [Row(_sig(L, 300 + i), cv=("volume", (v,)), delay=D, amp=0.3 + 0.05 * i, agc=AGC_ROWS[i % 2]) for i, (L, v) in enumerate(zip(lens, vols))]
    return Case("window_mono_cv_echo_agc", 1, rows)


def _window_stereo():
    """Stereo ChannelVolume (no Spatial) -> reverb (999 samples: odd) -> AGC: n_out just below / above 8192, n_in just below /
    above 8192, a long stream last in its CTA."""
    D = 999
    lens = [7192, 7194, 8190, 8194, 8192, 2, 6000, 20000]
    rows = [Row(_sig(L, 400 + i), cv=("volume", (0.9 - 0.1 * i, 0.4 + 0.15 * i)), delay=D, agc=AGC_ROWS[i % 2])
            for i, L in enumerate(lens)]
    return Case("window_stereo_cv_echo_agc", 2, rows)


def _echo_mono():
    """Mono reverb -> AGC, one delay per stream: 0; equal to the input; longer than the input; an empty input (the output is the
    echo's silence alone); delays 1000 .. 1003, which put n0 = delay + 8192, where the interior front path begins, on a group of
    four and 1, 2, 3 samples past one."""
    spec = [(501, 0), (1001, 1001), (301, 1001), (0, 999), (10001, 1000), (10001, 1001), (10003, 1002), (9999, 1003), (6001, 4097)]
    rows = [Row(_sig(L, 500 + i), delay=D, amp=0.5, agc=AGC_ROWS[i % 2]) for i, (L, D) in enumerate(spec)]
    return Case("echo_edges_mono", 1, rows)


def _echo_stereo():
    """Stereo Spatial -> reverb -> AGC -> limit: a delay equal to the input, longer (odd), over an empty input, odd and even delays
    on each side of a group of four at the interior edge, delay 0."""
    spec = [(600, 600), (200, 1201), (0, 7), (10002, 999), (10002, 1001), (10000, 8), (10000, 9), (6000, 0)]
    rows = [Row(_sig(L, 600 + i, 1.2), cv=("spatial", (float(i % 3 - 1), 1.0, 0.0)), delay=D, agc=AGC_ROWS[i % 2], lim=LIMITS[i % 8])
            for i, (L, D) in enumerate(spec)]
    return Case("echo_edges_stereo_agc_limit", 2, rows)


def _late_mono():
    """Late joiners in the default launch: the four streams of a CTA share a start, the CTAs do not -- later, earlier than the group
    listed before (the batch takes the streams in the mixer's insertion order, by start), and far beyond the end of every stream
    of other CTAs; the last CTA holds three streams."""
    rng = np.random.default_rng(7)
    starts = [0] * 4 + [777] * 4 + [20000] * 4 + [123] * 4 + [30001] * 3
    rows = []
    for i, s in enumerate(starts):
        n_out = 9003 if i == 9 else int(rng.integers(250, 1000)) * 4 + 1 + i % 3
        rows.append(Row(_sig(n_out - 17 - i, 700 + i), start=s, cv=("volume", (0.5 + 0.1 * (i % 7),)), delay=17 + i,
                        agc=AGC_ROWS[i % 2]))
    return Case("late_joiners_mono_cv_echo_agc", 1, rows, launches=("default",))


def _late_stereo():
    """Late joiners, stereo ChannelVolume -> limit (no AGC): CTAs of four starting at 0, 74 and 2000, and a last one of two streams
    that start after every other stream has ended (listed second)."""
    starts = [0] * 4 + [30000] * 2 + [74] * 4 + [2000] * 4
    rows = [Row(_stereo_lr(1500 + 301 * i, 800 + i, 2.0, 0.2), start=s, cv=("volume", (1.0, 0.5 + 0.1 * i)), lim=LIMITS[i % 8])
            for i, s in enumerate(starts)]
    return Case("late_joiners_stereo_cv_limit", 2, rows, launches=("default",))


def _starts_differ():
    """Starts that differ inside a group of four: k_fused_fx does not take the batch, the general path does, and must still be right."""
    starts = [0, 0, 0, 5, 100, 100, 300, 300]
    rows = [Row(_sig(2001 + 10 * i, 900 + i), start=s, delay=33, agc=AGC_DEFAULT) for i, s in enumerate(starts)]
    return Case("starts_differ_in_group", 1, rows, launches=("default",), family=-1)


def _limit_mono():
    """Mono ChannelVolume -> limit, one preset or threshold per stream, loud input."""
    rows = [Row(_sig(3001 + 502 * i, 1000 + i, 1.5), cv=("volume", (0.8 + 0.1 * i,)), lim=LIMITS[i]) for i in range(8)]
    return Case("limit_presets_mono_cv", 1, rows)


def _limit_stereo():
    """Stereo reverb -> limit: channels of different level that swap halfway, so that coupling the channels through the other
    channel's previous peak (limit.rs:946-960) matters."""
    rows = [Row(_stereo_lr(3000 + 250 * i, 1100 + i, 2.5, 0.05), delay=2 * i + 1, amp=0.3, lim=LIMITS[(i + 3) % 8]) for i in range(7)]
    return Case("limit_presets_stereo_echo", 2, rows)


def _agc_mono():
    """Mono AGC alone, per-row settings at the floor above the settled gain, absolute_max_gain, the 0.1 clamp and times cut to
    10 s, each held for more than one RMS window."""
    rows = [Row(_sig(12001 + 2 * i, 1200 + i, AGC_AMP[i % 6]), agc=AGC_ROWS[i % 6]) for i in range(10)]
    return Case("agc_settings_mono", 1, rows)


def _agc_limit_mono():
    """Mono AGC -> limit with per-row AGC settings and limiter presets."""
    rows = [Row(_sig(9001 + 4 * i, 1300 + i, AGC_AMP[i % 6]), agc=AGC_ROWS[i % 6], lim=LIMITS[i % 8]) for i in range(6)]
    return Case("agc_limit_mono", 1, rows)


def _agc_stereo():
    """Stereo Spatial -> AGC -> limit with per-row AGC settings and limiter presets."""
    rows = [Row(_sig(2 * (5000 + 3 * i), 1400 + i, AGC_AMP[i % 6]), cv=("spatial", (float(i - 3), 0.5, 0.0)), agc=AGC_ROWS[i % 6],
                lim=LIMITS[(i + 1) % 8]) for i in range(7)]
    return Case("agc_settings_stereo_spatial_limit", 2, rows)


def _burst_mono():
    """A loud burst, silence, then quiet input, in streams whose bursts differ (the residue the f32 running sum keeps differs in
    size and sign), beside a clean stream in each CTA."""
    rows = []
    for i in range(8):
        if i % 4 == 3:
            rows.append(Row(_sig(15001, 1500 + i), agc=AGC_DEFAULT))
            continue
        burst = 1500 + 500 * i
        x = _burst(1500 + i, 300.0 + 150.0 * i, burst, 9000, 4001)
        if i == 0:
            x[:burst] = np.where(np.arange(burst) % 3, 2.0, -2.0)      # squares of 4: every sum is exact, the residue is 0
        rows.append(Row(x, agc=AGC_BURST, branch=(burst + RMS_WINDOW, RESIDUE)))
    return Case("agc_burst_silence_mono", 1, rows)


def f32_residue(x, burst):
    """What the f32 running sum of agc.rs (sum - old) + new holds once the window has passed the burst (x silent behind it)."""
    F = np.float32
    ring, s = np.zeros(RMS_WINDOW, F), F(0.0)
    for n in range(burst + RMS_WINDOW):
        q = F(abs(x[n]) * abs(x[n]))
        s = F(F(s - ring[n % RMS_WINDOW]) + q)
        ring[n % RMS_WINDOW] = q
    return float(s)


def _burst_stereo():
    """The burst, stereo, behind reverb and in front of a limiter."""
    rows = []
    for i in range(6):
        burst = 2 * (800 + 300 * i)
        D = 2 * i + 1
        rows.append(Row(_burst(1600 + i, 3.0 + 9.0 * i, burst, 2 * 5000, 2 * 2001), delay=D, agc=AGC_DEFAULT, lim=LIMITS[i],
                        branch=(burst + D + RMS_WINDOW, RESIDUE)))
    return Case("agc_burst_silence_stereo", 2, rows)


def _overflow():
    """Samples of 1e20 (and 3e19 in a stream of its own), whose squares overflow the f32 sum to inf; clean streams beside them."""
    rows = []
    for i in range(6):
        x = _sig(12001 + 2 * i, 1700 + i)
        br = None
        if i in (1, 4):
            at = 2000 + 700 * i
            x[at:at + 40] = np.float32(1e20 if i == 1 else -3e19)
            br = (at, OVERFLOW)
        rows.append(Row(x, agc=AGC_ROWS[i % 2], branch=br))
    return Case("agc_overflowing_squares", 1, rows)


def _nonfinite_mono():
    """Isolated NaN, +Inf and -Inf samples, each in one stream of a CTA whose other streams are clean (the mixer sum of that CTA is
    NaN or infinite from there on), through the AGC."""
    rows = []
    spec = {1: (3000, np.nan, NAN_SUM), 6: (4001, np.inf, INF_SUM), 8: (2500, -np.inf, INF_SUM)}
    for i in range(10):
        x = _sig(11001 + 2 * i, 1800 + i)
        br = None
        if i in spec:
            at, v, why = spec[i]
            x[at] = np.float32(v)
            br = (at, why)
        rows.append(Row(x, agc=AGC_ROWS[i % 6], branch=br))
    return Case("agc_nonfinite_mono", 1, rows)


def _nonfinite_stereo():
    """NaN and +Inf in one stereo stream each, through ChannelVolume, reverb, AGC and the limiter (whose peak stays NaN, or whose
    integrator stays at +inf, for the rest of the stream)."""
    rows = []
    for i in range(6):
        x = _sig(2 * (5001 + i), 1900 + i)
        br = None
        if i in (1, 4):
            at = 2 * 1500 + 1 + 2 * i
            x[at] = np.float32(np.nan if i == 1 else np.inf)
            br = (at, NAN_SUM if i == 1 else INF_SUM)
        rows.append(Row(x, cv=("volume", (0.9, 1.1)), delay=101, agc=AGC_DEFAULT, lim=LIMITS[i], branch=br))
    return Case("agc_nonfinite_stereo_limit", 2, rows)


def _tiny():
    """Subnormal samples (whose squares underflow to 0 in f32), stretches of -0.0 and +0.0, a stream of -0.0 alone; AGC with no
    front stage, so that -0.0 reaches the streams' outputs."""
    rows = []
    for i in range(6):
        x = _sig(9001 + 2 * i, 2000 + i)
        if i == 1:
            x[:] = np.float32(-0.0)
        elif i in (2, 4):
            x[1000:3000] = noise(2000, 2100 + i, 1e-38) * np.float32(1e-3)
            x[5000:5100] = np.float32(-0.0)
            x[5100:5200] = np.float32(0.0)
            x[7000:9000] = np.float32(-1.4e-45)
        rows.append(Row(x.astype(np.float32), agc=AGC_ROWS[i % 3]))
    return Case("agc_subnormal_signed_zero", 1, rows)


def _two_waves():
    """1100 short stereo streams (275 CTAs: more than two waves of one CTA per SM) through Spatial -> reverb -> AGC: in exact order
    the ticket order and the tags cross waves, and come round again on the second render."""
    rng = np.random.default_rng(11)
    rows = [Row(_sig(2 * int(rng.integers(60, 400)), 3000 + i, 0.4), cv=("spatial", (float(i % 7 - 3), 1.0, 0.0)),
                delay=int(rng.integers(0, 40)), agc=AGC_DEFAULT) for i in range(1100)]
    return Case("exact_order_two_waves", 2, rows)


DESIGNS = [_short_mono, _short_stereo, _window_mono, _window_stereo, _echo_mono, _echo_stereo, _late_mono, _late_stereo,
           _starts_differ, _limit_mono, _limit_stereo, _agc_mono, _agc_limit_mono, _agc_stereo, _burst_mono, _burst_stereo,
           _overflow, _nonfinite_mono, _nonfinite_stereo, _tiny, _two_waves]
CASE_NAMES = [d().name for d in DESIGNS]


@functools.lru_cache(maxsize=None)
def build_case(name):
    return next(c for c in (d() for d in DESIGNS) if c.name == name)


@functools.lru_cache(maxsize=4)
def expected(name):
    """The oracle's per-stream outputs and sequential mix, the f64 streams, the f64 mix and its trusted positions."""
    case = build_case(name)
    srcs = case.sources()
    per_stream = [oracle.chain_uniform(to_oracle(s), case.ch, RATE) for s in srcs]
    ref = oracle.mixer([to_oracle(s, st) for s, st in zip(srcs, case.starts)], case.ch, RATE)
    ys = f64_streams(case)
    truth, trust = f64_mix(case, ys)
    return per_stream, ref, ys, truth, trust


# ------------------------------------------------------------------ GPU tests
GENERAL = capi.RB_KEEP_STREAM_OUTPUTS | capi.RB_NO_FUSION | capi.RB_MIX_EXACT_ORDER


def device_streams(ctx, case):
    """Every stream's output from the general path (one launch per adapter level): with a limiter, the per-stream samples
    k_fused_fx must reproduce bit for bit, because both take log2 / exp2 from the same device functions (within 2 ulp of
    glibc's, so not the oracle's bits)."""
    with rb.Batch(case.sources(), case.ch, RATE, flags=GENERAL, mix_starts=case.starts, ctx=ctx) as b:
        assert b.kernel_family == -1
        b.upload_all()
        b.render_mix()
        return [b.read_stream(i) for i in range(len(case.rows))]


def render(ctx, case, launch):
    """Mixer output of one launch, rendered twice (the second render must repeat the first bit for bit)."""
    flags = capi.RB_MIX_EXACT_ORDER if launch == "chain" else 0
    with rb.Batch(case.sources(), case.ch, RATE, flags=flags, mix_starts=case.starts, ctx=ctx) as b:
        family, group = b.kernel_family, b.mix_group
        b.upload_all()
        got = b.render_mix()
        again = b.render_mix()
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32)), f"{case.name} {launch}: render is not idempotent"
    return got, family, group


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_fx_rows(ctx, name):
    case = build_case(name)
    per_stream, ref, _, truth, trust = expected(name)
    assert truth.size == ref.size
    e_ref, peak = finite_distance(ref, truth, trust)
    if name == "exact_order_two_waves":
        assert -(-len(case.rows) // FX_R) > 2 * ctx.sm_count, "the chain must span more than two waves of CTAs"
    streams, source = per_stream, "oracle"
    if case.rows[0].lim is not None:
        streams, source = device_streams(ctx, case), "general-path"
        for i, (y, o) in enumerate(zip(streams, per_stream)):
            assert y.size == o.size and np.array_equal(np.isnan(y), np.isnan(o)), f"{name}: general-path stream {i}"
            e, p = finite_distance(y, o)
            assert e <= 1e-5 * p, f"{name}: general-path stream {i} is {e:.3e} from the oracle's, peak {p:.3e}"
    for launch in case.launches:
        got, family, group = render(ctx, case, launch)
        if launch == "chain":
            assert (family, group) == (5, 0), f"{name} chain: kernel family {family}, mix group {group}"
            if source == "oracle":
                assert_same(got, ref, f"{name}, exact-order chain vs the reference's sequential mixer")
            else:
                want = grouped_expected_mix(streams, case.starts, ref.size, len(streams))
                assert_same(got, want, f"{name}, exact-order chain vs the general path's streams summed in order")
                e, p = finite_distance(got, ref)
                assert e <= 1e-5 * p, f"{name} chain: {e:.3e} from the sequential mixer, peak {p:.3e}"
        else:
            assert family == case.family, f"{name}: kernel family {family}, expected {case.family}"
            if family == 5:
                assert group == FX_R, f"{name}: mix group {group}"
                want = grouped_expected_mix(streams, case.starts, ref.size)
                assert_same(got, want, f"{name}, default launch vs {source} streams added in the kernel's order")
            else:
                assert group == 0, f"{name}: mix group {group}"
                assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{name}: NaN masks differ from the sequential mixer"
            e, p = finite_distance(got, ref)
            assert e <= 1e-5 * p, f"{name} {launch}: {e:.3e} from the sequential mixer, peak {p:.3e}"
        e_got, _ = finite_distance(got, truth, trust)
        assert e_got <= F64_FACTOR * e_ref + 1e-7 * peak, f"{name} {launch}: {e_got:.3e} from the f64 mix, oracle {e_ref:.3e}"


# ------------------------------------------------------------------ CPU: the f64 restatement against the oracle, the designs
@pytest.mark.parametrize("name", CASE_NAMES)
def test_f64_restatement_matches_oracle(name):
    """On every design the oracle and the f64 restatement give every stream the same length, the same NaN and infinity masks,
    and stay within stream_tol of the stream's peak up to the listed branch point (if any); the oracle's mix stays within
    stream_tol of the f64 mix, and the oracle's streams added in k_fused_fx's order within the bound test_fx_rows applies."""
    case = build_case(name)
    per_stream, ref, ys, truth, trust = expected(name)
    for i, (r, y, t) in enumerate(zip(case.rows, per_stream, ys)):
        assert y.size == t.size == case.out_len(r), (i, y.size, t.size, case.out_len(r))
        for mask in (np.isnan, np.isposinf, np.isneginf):
            assert np.array_equal(mask(y), mask(t)), f"stream {i}: {mask.__name__} masks differ"
        upto = r.branch[0] if r.branch else y.size
        e, p = finite_distance(y[:upto], t[:upto])
        assert e <= stream_tol(y.size) * p + 1e-30, f"stream {i}: {e:.3e} from the f64 restatement, peak {p:.3e}"
    assert ref.size == truth.size
    e_ref, peak = finite_distance(ref, truth, trust)
    assert e_ref <= stream_tol(max(y.size for y in per_stream)) * peak, (e_ref, peak)
    if "default" in case.launches and case.family == 5:
        grouped = grouped_expected_mix(per_stream, case.starts, ref.size)
        e_grouped, _ = finite_distance(grouped, truth, trust)
        assert e_grouped <= 1.5 * e_ref + 1e-7 * peak, (e_grouped, e_ref, peak)


def test_designs_hold_the_edges():
    """The designs hold the edges the module docstring names, and every one fits k_fused_fx's planner (rb_fx_try_create) as
    intended: one node kind set per batch, equal starts inside each group of four unless the design is about the opposite."""
    cases = [build_case(n) for n in CASE_NAMES]
    mono = {r.pcm.size for c in cases if c.ch == 1 for r in c.rows}
    assert {0, 1, 3, 4, 5, TILE - 1, TILE, TILE + 1} <= mono
    n_out = {c.out_len(r) for c in cases for r in c.rows}
    assert {8191, 8193} <= n_out
    assert all(L % 4 for c in cases if c.ch == 1 and c.family == 5 for r in c.rows for L in [c.out_len(r)] if L > 300)
    echo = [(r.pcm.size, r.delay) for c in cases for r in c.rows if r.delay is not None]
    assert any(d == 0 for _, d in echo) and any(n == d for n, d in echo) and any(0 < n < d for n, d in echo)
    assert {d % 4 for n, d in echo if n > d + RMS_WINDOW} == {0, 1, 2, 3}
    assert any(d % 2 for c in cases if c.ch == 2 for r in c.rows for d in [r.delay or 0])
    last = {len(c.rows) % FX_R for c in cases if c.family == 5}
    assert {1, 2, 3} <= last
    for c in cases:
        kinds = {(r.cv is not None, r.delay is not None, r.agc is not None, r.lim is not None) for r in c.rows}
        assert len(kinds) == 1 and any(k[2] or k[3] for k in kinds), c.name
        starts = [c.rows[i].start for i in insertion_order(c.starts)]
        same = all(len(set(starts[g:g + FX_R])) == 1 for g in range(0, len(starts), FX_R))
        assert same == (c.family == 5), c.name
        if "chain" in c.launches:
            assert all(r.start == 0 for r in c.rows) and len(c.rows) > FX_R, c.name
        for i, r in enumerate(c.rows):
            if r.delay is not None:
                assert delay_samples(ns_for(r.delay, c.ch), c.ch) == r.delay
            assert r.start % c.ch == 0 and r.pcm.size % c.ch == 0, (c.name, i)
    shapes = {(c.ch, c.rows[0].cv[0] if c.rows[0].cv else None, c.rows[0].delay is not None, c.rows[0].agc is not None,
               c.rows[0].lim is not None) for c in cases}
    for ch in (1, 2):
        for back in ((True, False), (False, True), (True, True)):
            assert any(s[0] == ch and s[3:] == back for s in shapes), (ch, back)
        assert any(s[0] == ch and s[1] == "volume" for s in shapes)
    assert any(s[1] is None and s[2] is False for s in shapes)
    assert -(-len(build_case("exact_order_two_waves").rows) // FX_R) > 2 * H100_SMS
    residues = [f32_residue(r.pcm, r.branch[0] - RMS_WINDOW) for r in build_case("agc_burst_silence_mono").rows if r.branch]
    assert min(residues) < 0.0 and 0.0 in residues and max(residues) > 7.0, residues
