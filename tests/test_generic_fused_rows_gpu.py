"""k_fused_biquad and k_fused_nobiquad (kernel family 0) on batches whose rows differ inside one CTA.

Family 0 serves every fused-shape batch below 128 streams per SM that k_fused_hot cannot take: sources whose channel count is
not the mixer's, mixers of 3 to 12 channels, downsampling past the hot kernel's input window, SamplesBuffer clips whose
conversion restarts every 32 768 samples (ROW_GENERIC rows), batches that mix integer and f32 PCM (the F32 = false
instantiations), and filter-free chains of gains and channel maps.  The designs below put rows that differ in rate, channel
count, length, start, filter, gains, row mode and sample format into the same CTA, so that a row that reads another row's
parameters, a recurrence lane mapped to the wrong (row, channel), or a tile that cuts a frame at the wrong channel changes the
output.

Every design is checked on the device
  * for the kernel and launch it was built for: kernel family 0, the planner's rows per CTA, one launch for a single CTA and
    two otherwise;
  * bit for bit against the oracle's per-stream outputs added in the kernel's documented order (per CTA from +0.0 in the
    planner's stream order, the CTA partials in CTA order; NaN where the oracle has NaN, payloads not compared), twice;
  * against a float64 restatement of the chain written with numpy / scipy (format decode, channel map, chunked conversion, the
    biquad with the f32 coefficients every implementation uses), which must stay within twice the oracle's own distance.
The CPU tests pin the float64 restatement against the oracle and check, from the planner's rules, that every design reaches
the kernel paths it claims."""
import functools
import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np
import pytest
import scipy.signal

import oracle
import rodio_b200 as rb
from helpers import assert_bit_exact, noise, to_oracle
from rodio_b200 import capi
from test_bench_geometries_gpu import grouped_expected_mix
from test_hot_rows_gpu import F64_FACTOR, H100_SMS, TT, lerp64, out_frames, reduced

SPAN_CAP = 32768                # UniformSourceIterator restarts its conversion every min(span, 32768) samples (uniform.rs)
WSTRIDE = 320                   # k_fused_hot's input window per row (floats): a wider one sends the batch here
FORMATS = ("f32", "i16", "u16", "i8", "u8", "i32", "i24")
AUDIO = 1e6                     # f64 distances are taken where the f64 mix stays below this (huge operands are checked bit for bit)


@dataclass
class Row:
    pcm: np.ndarray
    c_in: int
    rate: int
    start: int                              # requested mix start in mixer samples (the planner rounds it up to a frame)
    fmt: str = "f32"
    span: int = 0                           # span_len the source reports (0: none, like TestSource; pcm.size: SamplesBuffer)
    pre: Tuple[float, ...] = ()             # gains in front of the conversion
    mid: Tuple[float, ...] = ()             # gains between the conversion and the filter
    filt: Optional[Tuple[bool, int, float]] = None   # (high pass?, frequency, q)
    post: Tuple[float, ...] = ()            # gains behind the filter
    conv: bool = True


@dataclass
class Case:
    name: str
    ch: int
    mix_rate: int
    rows: List[Row]                         # in the order they are handed to the mixer
    G: int                                  # rows per CTA the planner must choose
    filt: bool
    _f64: dict = field(default_factory=dict, repr=False)

    @functools.cached_property
    def order(self):
        """The planner's stream order: a stable sort by the requested start (Mixer::add order, ties in array order)."""
        return sorted(range(len(self.rows)), key=lambda i: self.rows[i].start)

    @functools.cached_property
    def kernel_rows(self):
        return [self.rows[i] for i in self.order]

    def frame_start(self, r):
        return -(-r.start // self.ch) * self.ch

    @functools.cached_property
    def starts(self):
        """Frame-aligned starts in the planner's order."""
        return [self.frame_start(r) for r in self.kernel_rows]

    def source(self, r):
        s = rb.Source(r.pcm, r.c_in, r.rate, span_len=r.span)
        if r.fmt == "i24":
            s.fmt_override = capi.RB_FMT_I24_IN_I32
        for g in r.pre:
            s = s.amplify(g)
        if r.conv:
            s = rb.UniformSourceIterator(s, self.ch, self.mix_rate)
        for g in r.mid:
            s = s.amplify(g)
        if r.filt:
            high, f, q = r.filt
            s = s.high_pass_with_q(f, q) if high else s.low_pass_with_q(f, q)
        for g in r.post:
            s = s.amplify(g)
        return s

    def stream64(self, k):
        """float64 restatement of the k-th stream in the planner's order (cached)."""
        if k not in self._f64:
            self._f64[k] = f64_stream(self.kernel_rows[k], self)
        return self._f64[k]

    def out_len(self, k):
        return self.stream64(k).size

    @property
    def n_ctas(self):
        return -(-len(self.rows) // self.G)

    def ctas(self):
        """(first row, rows) of every CTA, rows in the planner's order."""
        rows = self.kernel_rows
        return [(c * self.G, rows[c * self.G:(c + 1) * self.G]) for c in range(self.n_ctas)]

    @functools.cached_property
    def mix_len(self):
        return max(s + self.out_len(k) for k, s in enumerate(self.starts))


# ------------------------------------------------------------------ planner mirrors (rb_fused.cu, rb_fused_rows.h)
def rows_per_cta(sms, S, C, has_b):
    """G of rb_fused_try_create for a batch that is neither hot nor the lane kernels': up to 32 rows, with a filter at most
    128 (row, channel) chains (4 recurrence warps); one balanced wave over the SMs, k CTAs per SM beyond that."""
    max_g = 32
    while has_b and max_g > 1 and max_g * C > 128:
        max_g -= 1
    k = -(-S // (sms * max_g))
    G = -(-S // (sms * k))
    return max(1, min(G, max_g))


def grid_y(sms, n_ctas, mix_len):
    """k_fused_nobiquad's timeline slices: about eight CTAs per SM."""
    tiles = -(-mix_len // TT)
    return max(1, min(tiles, -(-sms * 8 // n_ctas), 65535))


def chunk_of(r):
    chunk = min(r.span, SPAN_CAP) if r.span else 0
    return 0 if chunk >= r.pcm.size else chunk


def row_mode(r, mix_rate):
    """parse_row's row mode: DIRECT (no conversion), PASS (same rate, whole-frame chunks), LERP (one chunk), GENERIC."""
    if not r.conv:
        return "direct"
    chunk = chunk_of(r)
    if reduced(r.rate, mix_rate)[0] == reduced(r.rate, mix_rate)[1]:
        return "pass" if chunk == 0 or chunk % r.c_in == 0 else "generic"
    return "lerp" if chunk == 0 else "generic"


def is_hot(case, sms):
    """Whether rb_fused_try_create would hand the batch to k_fused_hot (family 1) or the lane kernels instead."""
    C, rows = case.ch, case.rows
    has_u = any(r.conv for r in rows)
    all_f32 = all(r.fmt == "f32" for r in rows)
    if len(rows) >= 128 * sms:
        return True
    if not case.filt and has_u and C == 1 and len(rows) >= 64 and all_f32 and all(r.c_in == 1 for r in rows):
        return True                          # the timeline-segment plans of the lane kernels
    if not ((case.filt or has_u) and all_f32 and C in (1, 2)):
        return False
    for k, r in enumerate(case.kernel_rows):
        mode = row_mode(r, case.mix_rate)
        f, t = reduced(r.rate, case.mix_rate)
        qT = (TT // C) * f // t
        whole = r.pcm.size % C == 0 and case.out_len(k) % C == 0
        if not (r.c_in == C and whole and (mode in ("direct", "pass") or (mode == "lerp" and 3 + (qT + 3) * C <= WSTRIDE))):
            return False
        if not case.filt and mode != "lerp":
            return False
    return True


# ------------------------------------------------------------------ the float64 restatement
def decode64(pcm, fmt):
    """dasp_sample's X -> f32 conversions in float64 (the i32 value is rounded to f32 first, as `as f32` does)."""
    v = pcm.astype(np.float64)
    if fmt == "i32":
        return pcm.astype(np.float32).astype(np.float64) / 2.0 ** 31
    return {"f32": v, "i16": v / 32768.0, "u16": (v - 32768.0) / 32768.0, "i8": v / 128.0, "u8": (v - 128.0) / 128.0,
            "i24": v / 2.0 ** 23}[fmt]


def chan_map(j, c_in):
    """channels.rs: output channel j reads input channel j, a mono source feeds channel 1 as well, the rest is 0."""
    return j if j < c_in else (0 if j == 1 and c_in == 1 else -1)


def map_channels(flat, c_in, C):
    """ChannelCountConverter over a flat run: whole frames, then the channels of a trailing partial frame that exist."""
    groups, k = divmod(flat.size, c_in)
    out = np.zeros(groups * C + min(k, C), dtype=np.float64)
    frames = flat[:groups * c_in].reshape(groups, c_in)
    for j in range(C):
        c = chan_map(j, c_in)
        if c >= 0:
            out[j:groups * C:C] = frames[:, c]
    for j in range(min(k, C)):
        out[groups * C + j] = flat[groups * c_in + chan_map(j, c_in)]
    return out


def f64_stream(r, case):
    gain = lambda v: float(np.float32(v))
    x = decode64(r.pcm, r.fmt)
    for g in r.pre:
        x = x * gain(g)
    if r.conv:
        chunk = chunk_of(r)
        pieces = [x[i:i + chunk] for i in range(0, x.size, chunk)] if chunk else [x]
        out = []
        for p in pieces:                    # every chunk converted on its own, its last frame raw
            f, t = reduced(r.rate, case.mix_rate)
            if f != t:
                assert p.size % r.c_in == 0, "resampled chunks of whole frames only"
                with np.errstate(all="ignore"):     # Inf and NaN operands
                    p = lerp64(p.reshape(-1, r.c_in), r.rate, case.mix_rate).reshape(-1)
            out.append(map_channels(p, r.c_in, case.ch))
        x = np.concatenate(out)
    for g in r.mid:
        x = x * gain(g)
    if r.filt and x.size:
        high, f, q = r.filt
        b0, b1, b2, a1, a2 = (float(v) for v in oracle.blt_coeffs(high, f, q, case.mix_rate))
        x = x.copy()
        with np.errstate(all="ignore"):
            for c in range(case.ch):        # one filter state per channel, by position in the interleaved stream
                x[c::case.ch] = scipy.signal.lfilter([b0, b1, b2], [1.0, a1, a2], x[c::case.ch])
    for g in r.post:
        x = x * gain(g)
    return x


def f64_mix(case):
    total = np.zeros(case.mix_len, dtype=np.float64)
    with np.errstate(all="ignore"):
        for k, s in enumerate(case.starts):
            y = case.stream64(k)
            total[s:s + y.size] += y
    return total


# ------------------------------------------------------------------ designed batches
def _gains(rng, n):
    return tuple(float(np.float32(0.4 + 1.2 * rng.random())) for _ in range(n))


def _filter(rng, mix_rate):
    return (bool(rng.random() < 0.3), int(rng.integers(100, int(0.35 * mix_rate))), float(np.float32(0.4 + 0.8 * rng.random())))


def pcm_of(fmt, n, seed):
    x = noise(n, seed).astype(np.float64)
    return {"f32": lambda: x.astype(np.float32),
            "i16": lambda: np.round(x * 32767).astype(np.int16),
            "u16": lambda: (np.round(x * 32767) + 32768).astype(np.uint16),
            "i8": lambda: np.round(x * 127).astype(np.int8),
            "u8": lambda: (np.round(x * 127) + 128).astype(np.uint8),
            "i32": lambda: np.round(x * 2147483000.0).astype(np.int32),
            "i24": lambda: np.round(x * 8388607.0).astype(np.int32)}[fmt]()


@dataclass
class Kind:
    c_in: int
    rate: int
    fmt: str = "f32"
    span: int = 0                       # -1: the whole clip (SamplesBuffer)
    frames: Optional[Tuple[int, int]] = None   # input frames drawn from [lo, hi] (default: the design's range)


def designed(name, sms, S, C, kinds, *, mix_rate=48000, seed=0, filt=True, n_pre=0, n_mid=1, n_post=1, conv=True,
             frames=(300, 900), cta_span=1024, edges=False, shuffle=False, unaligned=False, chunk_at_tile=False):
    """S rows, CTA after CTA (G rows each, as the planner will cut them).  Row g of CTA c is of kind (c + g) % len(kinds), so
    every CTA of at least len(kinds) rows holds every kind; starts are spread over the first half of the CTA's `cta_span`
    frames, and every row has its own length, filter and gains.
    edges: CTA 0 only empty rows, CTA 1 rows of 0, 1 and 2 frames beside full ones, CTA 2 and the last two CTAs a row that
    starts after every other row of its CTA has ended.
    unaligned: requested starts up to C - 1 samples before a frame (the planner rounds them up); shuffle: the rows are handed
    over in random order (the planner sorts them back by requested start, ties in hand-over order).
    chunk_at_tile: rows with span restarts start where their first restart lands on a tile boundary (every other one)."""
    rng = np.random.default_rng(seed)
    G = rows_per_cta(sms, S, C, filt)
    rows = []
    n_ctas = -(-S // G)
    for c in range(n_ctas):
        n = min(G, S - c * G)
        late = edges and c in (2, n_ctas - 2, n_ctas - 1) and n > 1
        cta = []
        for g in range(n):
            kd = kinds[(c + g) % len(kinds)]
            lo, hi = kd.frames or frames
            L = int(rng.integers(lo, hi + 1))
            off = int(rng.integers(0, cta_span // 2))
            if edges and c == 0:
                L = 0
            elif edges and c == 1 and g < 3:
                L = g
            elif late:
                L = min(L, 60)
                off = min(off, 100)
                if g == n - 1:
                    off = cta_span - 1
            pcm = pcm_of(kd.fmt, L * kd.c_in, seed * 100003 + c * 131 + g)
            span = pcm.size if kd.span == -1 else kd.span
            start = (c * cta_span + off) * C
            r = Row(pcm, kd.c_in, kd.rate, start, kd.fmt, span, _gains(rng, n_pre), _gains(rng, n_mid),
                    _filter(rng, mix_rate) if filt else None, _gains(rng, n_post), conv)
            if chunk_at_tile and g % 2 == 0 and chunk_of(r):
                full_out = out_frames(SPAN_CAP // kd.c_in, kd.rate, mix_rate) * C
                base = c * cta_span * C
                r.start = base + (-(base + full_out)) % TT          # the first restart lands on a tile boundary
                assert r.start % C == 0 and r.start < base + cta_span * C // 2
            cta.append(r)
        cta.sort(key=lambda r: r.start)
        rows += cta
    if unaligned:
        for r in rows:
            d = int(rng.integers(0, C))
            if r.start >= d:
                r.start -= d
    if shuffle:
        rows = [rows[i] for i in rng.permutation(len(rows))]
    return Case(name, C, mix_rate, rows, G, filt)


def _plant_operands(case, seed, nan_inf=True):
    """Operands outside lerp_rcp's exact-reciprocal range in one f32 row of each multi-row CTA, in the middle of the row:
    denormal differences, +-3e30, +-Inf, NaN, signed zeros (by CTA); in 2:1 rows an Inf on a right tap only (num = 0: the
    reference's (Inf - a) * 0 is NaN).  nan_inf=False: only the finite kinds (rows behind a filter)."""
    rng = np.random.default_rng(seed)
    kinds = ("denormal", "huge", "inf", "ninf", "nan", "zeros") if nan_inf else ("denormal", "huge", "zeros")
    for c, (_, rows) in enumerate(case.ctas()):
        cand = [r for r in rows if r.fmt == "f32" and r.pcm.size >= 64 * r.c_in]
        if len(rows) < 2 or not cand:
            continue
        r = cand[int(rng.integers(len(cand)))]
        i = r.pcm.size // 2 // r.c_in * r.c_in
        kind = kinds[c % len(kinds)]
        vals = {"denormal": list(noise(6, c) * np.float32(1e-38)), "huge": [3e30, -3e30, 1.0, 3e30],
                "inf": [np.inf], "ninf": [-np.inf], "nan": [np.nan], "zeros": [0.0, -0.0, -0.0, 0.0, -0.0]}[kind]
        r.pcm[i:i + len(vals)] = np.asarray(vals, dtype=np.float32)
        two = [q for q in rows if q.fmt == "f32" and reduced(q.rate, case.mix_rate) == (2, 1) and q.c_in == 1 and q.pcm.size > 40]
        if nan_inf and two:
            two[0].pcm[2 * 7 + 1] = np.float32(np.inf)    # frame 7's right tap; frame 8's left tap is x[16]
    return case


K = Kind
STEREO_KINDS = [K(1, 44100), K(2, 44100), K(1, 32000), K(2, 22050), K(1, 96000), K(2, 88200), K(1, 192000), K(1, 48000)]
FMT_RATES = (44100, 32000, 96000, 22050, 88200, 44100, 32000)


def _format_kinds(stereo):
    return [K(2 if stereo and i % 2 else 1, FMT_RATES[i], f) for i, f in enumerate(FORMATS)]


def _cases(sms):
    return {
        # 1. stereo mixer, mono and stereo sources, 2:1 and steeper: 32 rows (64 chains, 2 recurrence warps), the last CTA 31
        "stereo_mono_g32": lambda: designed("stereo_mono_g32", sms, 32 * sms - 1, 2, STEREO_KINDS, seed=1),
        "stereo_mono_g3": lambda: designed("stereo_mono_g3", sms, 2 * sms + 40, 2, STEREO_KINDS, seed=2, n_pre=1),
        # 2. surround mixers at max_g: mono, stereo, the mixer's own count (another rate) and one more (dropped channels);
        #    partial last CTAs of 30, 65, 102 and 36 chains
        "surround3_g32": lambda: designed("surround3_g32", sms, 32 * sms - 22, 3,
                                          [K(1, 44100), K(2, 32000), K(3, 44100), K(4, 48000), K(1, 48000), K(3, 22050),
                                           K(2, 96000), K(4, 44100)], seed=3, frames=(150, 500)),
        "surround5_g25": lambda: designed("surround5_g25", sms, 25 * sms - 12, 5,
                                          [K(1, 44100), K(2, 48000), K(5, 32000), K(6, 44100), K(5, 96000), K(2, 22050)],
                                          seed=4, frames=(150, 400)),
        "surround6_g21": lambda: designed("surround6_g21", sms, 21 * sms - 4, 6,
                                          [K(1, 48000), K(2, 44100), K(6, 44100), K(7, 88200), K(1, 32000), K(2, 48000)],
                                          seed=5, frames=(150, 400), n_mid=0, n_post=2),
        "surround12_g10": lambda: designed("surround12_g10", sms, 10 * sms - 7, 12,
                                           [K(1, 44100), K(2, 48000), K(12, 32000), K(11, 48000), K(12, 96000)],
                                           seed=6, frames=(100, 300)),
        # 3. mono mixer at 8 kHz: 96 k, 88.2 k, 192 k, 48 k and 44.1 k rows in one CTA (windows far past k_fused_hot's)
        "mono_steep_8k": lambda: designed("mono_steep_8k", sms, 32 * sms - 9, 1,
                                          [K(1, 96000, frames=(1200, 4800)), K(1, 88200, frames=(1100, 4400)),
                                           K(1, 192000, frames=(2400, 9600)), K(1, 44100, frames=(550, 2200)),
                                           K(1, 48000, frames=(600, 2400))], mix_rate=8000, seed=7, cta_span=512),
        # 4. span restarts: SamplesBuffer clips of 32768 +- a few samples and of more than two chunks beside TestSource rows;
        #    the first restart on a tile boundary for every other clip; a same-rate stereo clip of odd span into a mono mixer
        "span_stereo": lambda: designed("span_stereo", sms, 3 * sms, 2,
                                        [K(1, 44100, span=-1, frames=(32765, 32771)), K(2, 44100),
                                         K(2, 44100, span=-1, frames=(16382, 16386)), K(1, 44100, span=-1, frames=(81920, 82000)),
                                         K(1, 32000), K(2, 22050, span=-1, frames=(49000, 49200))],
                                        seed=8, chunk_at_tile=True),
        "span_mono": lambda: designed("span_mono", sms, 3 * sms, 1,
                                      [K(1, 44100, span=-1, frames=(32765, 32771)), K(2, 44100, span=-1, frames=(16382, 16386)),
                                       K(1, 44100), K(2, 48000, span=1001, frames=(2900, 3100)),
                                       K(1, 22050, span=-1, frames=(81920, 82000)), K(2, 32000)],
                                      seed=9, n_pre=1, chunk_at_tile=True),
        "small_span_22k": lambda: designed("small_span_22k", sms, 2 * sms + 5, 2,
                                           [K(1, 44100, span=1024, frames=(9000, 10000)), K(2, 44100, span=1000, frames=(2000, 3000)),
                                            K(1, 32000), K(3, 44100, span=999, frames=(1500, 2500))],
                                           mix_rate=22050, seed=10),
        # 5. every sample format beside f32 rows in each 8-row CTA (F32 = false), with and without a filter
        "formats_mono": lambda: designed("formats_mono", sms, 8 * sms - 3, 1, _format_kinds(False), seed=11, n_pre=1),
        "formats_stereo": lambda: designed("formats_stereo", sms, 8 * sms - 3, 2, _format_kinds(True), seed=12),
        "formats_mono_nofilter": lambda: designed("formats_mono_nofilter", sms, 8 * sms - 3, 1, _format_kinds(False), seed=13,
                                                  filt=False, n_mid=2, n_post=0),
        "formats_stereo_nofilter": lambda: designed("formats_stereo_nofilter", sms, 8 * sms - 3, 2, _format_kinds(True),
                                                    seed=14, filt=False, n_pre=1, n_mid=1, n_post=0),
        # 6. k_fused_nobiquad: same-rate rows with 4 and 1 gains, channel maps with 3 and 2; a timeline cut over gridDim.y
        "nobiquad_direct_4gains": lambda: designed("nobiquad_direct_4gains", sms, 40, 2,
                                                   [K(2, 48000), K(2, 48000, "i16"), K(2, 48000, "u8")], seed=15, filt=False,
                                                   conv=False, n_pre=4, n_mid=0, n_post=0),
        "nobiquad_direct_g32": lambda: designed("nobiquad_direct_g32", sms, 32 * sms - 1, 1, [K(1, 48000)], seed=16, filt=False,
                                                conv=False, n_pre=1, n_mid=0, n_post=0),
        "nobiquad_chanmap_g32": lambda: designed("nobiquad_chanmap_g32", sms, 32 * sms - 2, 2,
                                                 [K(1, 48000), K(3, 48000), K(4, 48000), K(6, 48000)], seed=17, filt=False,
                                                 n_pre=1, n_mid=2, n_post=0),
        "nobiquad_chanmap_mono": lambda: designed("nobiquad_chanmap_mono", sms, 24, 1,
                                                  [K(2, 48000), K(3, 48000, "i16"), K(6, 48000)], seed=18, filt=False,
                                                  n_pre=2, n_mid=0, n_post=0),
        # 7. edges in every kernel: empty and one-frame rows, a CTA of empty rows, rows that start after their CTA ended,
        #    unaligned starts handed over out of order; single-stream batches (one CTA, written in place)
        "edges_mono": lambda: designed("edges_mono", sms, 4 * sms + 3, 1,
                                       [K(1, 44100), K(1, 32000), K(1, 96000), K(2, 44100), K(1, 22050)],
                                       seed=19, edges=True, shuffle=True),
        "edges_surround5": lambda: designed("edges_surround5", sms, 4 * sms + 3, 5,
                                            [K(1, 44100), K(2, 32000), K(5, 22050), K(6, 48000), K(5, 88200)],
                                            seed=20, edges=True, shuffle=True, unaligned=True),
        "edges_nobiquad": lambda: designed("edges_nobiquad", sms, 4 * sms + 3, 3,
                                           [K(1, 44100), K(3, 32000), K(2, 48000), K(4, 96000), K(3, 44100, "i16")],
                                           seed=21, filt=False, edges=True, shuffle=True, unaligned=True, n_mid=1, n_post=0),
        "single_biquad_mono": lambda: designed("single_biquad_mono", sms, 1, 1,
                                               [K(1, 44100, span=-1, frames=(40000, 40000))], seed=22),
        "single_biquad_c3": lambda: designed("single_biquad_c3", sms, 1, 3, [K(2, 32000, frames=(3000, 3000))], seed=23),
        "single_nobiquad": lambda: designed("single_nobiquad", sms, 1, 2, [K(1, 48000, "i16", frames=(5000, 5000))], seed=24,
                                            filt=False, n_mid=1, n_post=0),
        # 8. operands outside the exact-reciprocal range in one row of multi-row CTAs: stage_a_mono_lerp<false>,
        #    row_stage_a_any<false> (filter-free), and behind a filter (finite kinds only)
        "operands_mono": lambda: _plant_operands(designed("operands_mono", sms, 4 * sms, 1,
                                                          [K(1, 44100), K(1, 32000, "i16"), K(1, 96000), K(1, 22050)],
                                                          seed=25, filt=False, n_pre=1, n_mid=1, n_post=0), 25),
        "operands_stereo": lambda: _plant_operands(designed("operands_stereo", sms, 4 * sms, 2,
                                                            [K(1, 44100), K(2, 32000), K(1, 96000), K(1, 22050, "i16")],
                                                            seed=26, filt=False, n_mid=1, n_post=0), 26),
        "operands_filter": lambda: _plant_operands(designed("operands_filter", sms, 4 * sms, 2,
                                                            [K(1, 44100), K(2, 32000), K(1, 96000), K(1, 22050, "i16")],
                                                            seed=27), 27, nan_inf=False),
    }


CASE_NAMES = list(_cases(H100_SMS))


@functools.lru_cache(maxsize=2)
def build_case(name, sms):
    return _cases(sms)[name]()


def assert_same_mix(got, want, what):
    """Bit for bit, except that a NaN only has to meet a NaN (payloads are not compared)."""
    assert got.shape == want.shape, f"{what}: length {got.shape} != {want.shape}"
    gn, wn = np.isnan(got), np.isnan(want)
    bad = np.nonzero(gn != wn)[0]
    assert bad.size == 0, f"{what}: NaN masks differ at {bad.size} samples, first at {bad[0]}: got {got[bad[0]]!r} want {want[bad[0]]!r}"
    assert_bit_exact(np.where(gn, np.float32(0), got), np.where(wn, np.float32(0), want), what)


def f64_distance(y, truth):
    """max |y - truth| and the peak of truth, over the samples where both are finite and truth is audio-sized."""
    with np.errstate(all="ignore"):
        m = np.isfinite(truth) & np.isfinite(y) & (np.abs(truth) < AUDIO)
        if not m.any():
            return 0.0, 0.0
        return float(np.max(np.abs(y[m] - truth[m]))), float(np.max(np.abs(truth[m])))


# ------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_generic_fused_rows(ctx, name):
    case = build_case(name, ctx.sm_count)
    srcs = [case.source(r) for r in case.kernel_rows]
    starts = case.starts
    per_stream = [oracle.chain_uniform(to_oracle(s), case.ch, case.mix_rate) for s in srcs]
    mix_len = max(s + y.size for s, y in zip(starts, per_stream))
    with rb.Batch([case.source(r) for r in case.rows], case.ch, case.mix_rate, mix_starts=[r.start for r in case.rows],
                  ctx=ctx) as b:
        assert b.kernel_family == 0, f"{name}: kernel family {b.kernel_family}"
        assert b.mix_group == case.G, f"{name}: {b.mix_group} rows per CTA, expected {case.G}"
        assert b.launches_per_render == (1 if case.n_ctas == 1 else 2), f"{name}: {b.launches_per_render} launches"
        assert b.mix_len == mix_len
        b.upload_all()
        got = b.render_mix()
        again = b.render_mix()
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32)), f"{name}: render is not idempotent"
    want = grouped_expected_mix(per_stream, starts, mix_len, case.G)
    assert_same_mix(got, want, f"{name}: family 0 vs oracle streams added in the kernel's order")
    ref = oracle.mixer([to_oracle(s, st) for s, st in zip(srcs, starts)], case.ch, case.mix_rate)
    truth = f64_mix(case)
    assert truth.size == ref.size == got.size
    e_ref, peak = f64_distance(ref, truth)
    e_got, _ = f64_distance(got, truth)
    assert e_got <= F64_FACTOR * e_ref + 1e-7 * peak, f"{name}: {e_got:.3e} from the f64 chain, reference {e_ref:.3e}"


# ------------------------------------------------------------------ CPU: the reference and the designs
@pytest.mark.parametrize("name", CASE_NAMES)
def test_f64_reference_matches_oracle(name):
    """The float64 restatement agrees with the oracle on every design: the same length for every stream, the same NaN and Inf
    positions, within 1e-4 of the stream's peak; and the oracle's streams added in the kernel's order stay within the bound
    test_generic_fused_rows applies.  Where they may part (listed): an i32 sample is rounded to f32 before its scaling in
    both; a NaN or Inf operand poisons a filtered row in both; huge operands are left to the bit-exact device check."""
    case = build_case(name, H100_SMS)
    srcs = [case.source(r) for r in case.kernel_rows]
    per_stream = [oracle.chain_uniform(to_oracle(s), case.ch, case.mix_rate) for s in srcs]
    for k, y in enumerate(per_stream):
        t = case.stream64(k)
        assert y.size == t.size, (name, k, y.size, t.size)
        with np.errstate(all="ignore"):
            assert np.array_equal(np.isnan(y), np.isnan(t)), (name, k, "NaN positions")
            assert np.array_equal(np.isinf(y), np.isinf(t)), (name, k, "Inf positions")
        e, peak = f64_distance(y, t)
        assert e <= 1e-4 * peak + 1e-30, (name, k, e, peak)
    ref = oracle.mixer([to_oracle(s, st) for s, st in zip(srcs, case.starts)], case.ch, case.mix_rate)
    truth = f64_mix(case)
    assert truth.size == ref.size == case.mix_len
    e_ref, peak = f64_distance(ref, truth)
    assert e_ref <= 1e-4 * peak, (e_ref, peak)
    grouped = grouped_expected_mix(per_stream, case.starts, ref.size, case.G)
    e_grouped, _ = f64_distance(grouped, truth)
    assert e_grouped <= 1.5 * e_ref + 1e-7 * peak, (e_grouped, e_ref, peak)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_design_stays_in_family_0(name):
    """Every row converts or none does (a dropped identity conversion would send the batch to the general path), the batch is
    not one for k_fused_hot or the lane kernels, and the designed CTAs are the planner's."""
    case = build_case(name, H100_SMS)
    for r in case.rows:
        identity = r.c_in == case.ch and reduced(r.rate, case.mix_rate)[0] == reduced(r.rate, case.mix_rate)[1]
        assert r.conv != identity, (name, r.c_in, r.rate)
        assert r.conv or (r.c_in == case.ch and r.rate == case.mix_rate)
    assert not is_hot(case, H100_SMS), name
    assert case.G == rows_per_cta(H100_SMS, len(case.rows), case.ch, case.filt)
    assert len({(len(r.pre), len(r.mid), len(r.post), r.filt is None) for r in case.rows}) == 1


def _tiles(case):
    """(cta, row index in CTA, row, m0, lo_t, hi_t) for every (row, tile) the kernels walk."""
    out = []
    for c, (first, rows) in enumerate(case.ctas()):
        for g, r in enumerate(rows):
            s, n = case.starts[first + g], case.out_len(first + g)
            for m0 in range(s // TT * TT, s + n, TT):
                out.append((c, g, r, m0, max(s, m0) - m0, min(s + n, m0 + TT) - m0))
    return out


def test_designs_reach_the_recurrence_mappings():
    """CTAs with 2, 3 and 4 recurrence warps; per-CTA chain counts just below and above 32, 64 and 96; tiles that cut a frame
    for C = 3, 5, 6, 12 at every phase (m0 + lo_t) % C can take (multiples of gcd(TT, C): rows start on a frame); mono rows whose first and last tiles leave head and tail residues
    1 to 3 in the 16-byte-aligned recurrence."""
    warps, chains = set(), set()
    phases = {}
    heads, tails = set(), set()
    for name in CASE_NAMES:
        case = build_case(name, H100_SMS)
        if not case.filt:
            continue
        warps.add(-(-case.G * case.ch // 32))
        ctas = case.ctas()
        chains |= {len(rows) * case.ch for _, rows in ctas}
        for c, g, r, m0, lo, hi in _tiles(case):
            if case.ch > 1 and len(ctas[c][1]) > 1:
                phases.setdefault(case.ch, set()).add((m0 + lo) % case.ch)
            if case.ch == 1 and len(ctas[c][1]) > 1 and hi > lo:
                heads.add(lo % 4)
                tails.add(hi % 4)
    assert {2, 3, 4} <= warps, warps
    for a, b in ((24, 32), (32, 40), (56, 64), (64, 72), (88, 96), (96, 104)):
        assert any(a < n <= b for n in chains), (a, b, sorted(chains))
    for C in (3, 5, 6, 12):
        assert TT % C and phases.get(C) == set(range(0, C, math.gcd(TT, C))), (C, phases.get(C))
    assert {1, 2, 3} <= heads and {1, 2, 3} <= tails, (heads, tails)


def test_designs_restart_conversions_inside_rows():
    """Rows with span restarts (ROW_GENERIC) beside LERP and PASS rows in the same CTA, restarts on a tile boundary and inside a
    tile, clips of 32768 +- a few samples (one chunk and two), of more than two chunks, and the odd-span pass-through."""
    at_tile = inside = 0
    modes_together = False
    sizes = set()
    odd_generic = False
    for name in ("span_stereo", "span_mono", "small_span_22k"):
        case = build_case(name, H100_SMS)
        for first, rows in case.ctas():
            modes = {row_mode(r, case.mix_rate) for r in rows}
            modes_together |= "generic" in modes and "lerp" in modes
            for g, r in enumerate(rows):
                chunk = chunk_of(r)
                if r.span and r.span != r.pcm.size:
                    odd_generic |= r.span % 2 == 1 and row_mode(r, case.mix_rate) == "generic" and r.rate == case.mix_rate
                if r.span == r.pcm.size:
                    sizes.add(r.pcm.size)
                if not chunk or chunk % r.c_in:
                    continue
                full_out = out_frames(chunk // r.c_in, r.rate, case.mix_rate) * case.ch
                s, n = case.starts[first + g], case.out_len(first + g)
                for k in range(1, r.pcm.size // chunk + 1):
                    pos = s + k * full_out
                    if pos < s + n:
                        at_tile += pos % TT == 0
                        inside += pos % TT != 0
    assert modes_together and odd_generic
    assert at_tile >= 20 and inside >= 20, (at_tile, inside)
    assert any(SPAN_CAP - 4 <= n < SPAN_CAP for n in sizes) and any(SPAN_CAP < n <= SPAN_CAP + 4 for n in sizes)
    assert any(n > 2 * SPAN_CAP for n in sizes)


def test_designs_mix_formats_in_one_cta():
    """Each integer format shares a CTA with f32 rows (the F32 = false instantiations), mono and stereo, with and without a
    filter; the all-integer batch would take the resident f32 copy instead."""
    for name in ("formats_mono", "formats_stereo", "formats_mono_nofilter", "formats_stereo_nofilter"):
        case = build_case(name, H100_SMS)
        assert any(r.fmt != "f32" for r in case.rows) and any(r.fmt == "f32" for r in case.rows)
        full = [rows for _, rows in case.ctas() if {r.fmt for r in rows} == set(FORMATS)]
        assert len(full) >= case.n_ctas - 2, (name, len(full), case.n_ctas)
        if case.ch == 2:
            assert any({r.c_in for r in rows} == {1, 2} for rows in full)


def test_nobiquad_designs_cut_the_timeline():
    """k_fused_nobiquad designs spread each CTA's timeline over gridDim.y > 1, at G = 1 and at G = 32, and use 1 to 4 gains."""
    gs, gains = set(), set()
    for name in CASE_NAMES:
        case = build_case(name, H100_SMS)
        if case.filt or case.n_ctas == 1:
            continue
        assert grid_y(H100_SMS, case.n_ctas, case.mix_len) > 1, name
        gs.add(case.G)
        r = case.rows[0]
        gains.add(len(r.pre) + len(r.mid))
    assert {1, 32} <= gs and {1, 2, 3, 4} <= gains, (gs, gains)


def test_edge_designs():
    """Empty and one-frame rows, a CTA of empty rows, a row that starts a tile or more after every other row of its CTA has
    ended, unaligned starts handed over out of order (the planner's sort is not the hand-over order), in each kernel; and
    single-stream batches written in place."""
    for name in ("edges_mono", "edges_surround5", "edges_nobiquad"):
        case = build_case(name, H100_SMS)
        lens = [case.out_len(k) for k in range(len(case.rows))]
        assert 0 in lens and any(0 < n <= case.ch * 2 for n in lens)
        ctas = case.ctas()
        assert any(all(case.out_len(f + g) == 0 for g in range(len(rows))) for f, rows in ctas)
        late = 0
        for f, rows in ctas:
            ends = [case.starts[f + g] + case.out_len(f + g) for g in range(len(rows) - 1) if case.out_len(f + g)]
            if ends and case.starts[f + len(rows) - 1] >= (max(ends) // TT + 1) * TT:
                late += 1
        assert late >= 2, name
        assert case.order != sorted(case.order)
        if case.ch > 1:
            assert any(r.start % case.ch for r in case.rows)
    for name in ("single_biquad_mono", "single_biquad_c3", "single_nobiquad"):
        assert build_case(name, H100_SMS).n_ctas == 1
