"""k_fused_hot on batches whose rows differ: rates, starts, lengths, filters and gains change from row to row, so that a row that
borrows another row's parameters, or a row map that drops or repeats a row, changes the output.

Stage A of the mono kernel walks a warp's two rows in one pass when their tiles are in phase (hot_stage_a_pair: both interior,
the same rate pair, the same r0) and one after the other otherwise.  The batches below are designed so that the first and second
rows of a warp meet in every relation: in phase with the same input frame, in phase with frames a multiple of `to` apart, the
same rate with another r0, another rate, one of the two in a partial, ended or not yet started tile.  Default launches (row map
21 + 11) and exact-order chains (RB_MIX_EXACT_ORDER, row map 23 + 9) pair the rows differently; both run.

Every case is checked three ways:
  * bit for bit: the default launch against the oracle's per-stream outputs added in the kernel's documented order (per CTA
    from +0.0, then the CTA partials in CTA order), the chain against the reference's sequential mixer;
  * against a float64 restatement of the chain written here with numpy / scipy (lerp on the reduced rate grid from exact
    integer indices, gains, the biquad in f64, the sum), which shares no code with the oracle -- only the filter coefficients,
    which are the f32 values every implementation uses;
  * coverage: the same batch on an instrumented build (-DRB_HOT_PATHS) counts row-tiles per stage-A outcome, so that a case
    cannot pass on the solo path alone, and the row-tile total proves every row was walked exactly once per tile.
The CPU tests at the end pin the float64 reference against the oracle and check the designs without a device."""
import contextlib
import functools
import json
import math
import os
import subprocess
import sys
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import pytest
import scipy.signal

import oracle
import rodio_b200 as rb
from helpers import assert_bit_exact, noise, to_oracle
from rodio_b200 import capi
from test_bench_geometries_gpu import grouped_expected_mix

TT = 256                        # mixer samples per tile (rb_fused_rows.h)
H100_SMS = 132                  # the SM count the CPU tests design for
PATHS = ("pair", "pair_failed", "solo", "redo", "strided")    # rb_fused.cu HOT_PATH_*, in order
# f64 bound: the kernel may be at most this many times further from the f64 chain than the reference's sequential mixer
# (plus 1e-7 * peak).  The kernel adds the same per-stream samples in another order (per CTA, then the CTA partials), which on
# these batches keeps it within 1.5x of the reference's own distance (test_f64_reference_matches_oracle pins that on the CPU).
F64_FACTOR = 2.0
OFFSETS = (0, 0, 0, 37, 147, 160, 197, 320, 441, 480, 517, 800)   # frames a second row starts after its CTA's first rows
CTA_SPAN = 1024                 # frames between the first rows of consecutive CTAs (starts stay sorted across the batch)
RATES_A = (44100, 44100, 44100, 32000, 22050)


@dataclass
class Row:
    pcm: np.ndarray
    rate: int
    start: int                  # mixer samples
    pre: Tuple[float, ...] = ()   # gains in front of the conversion
    mid: Tuple[float, ...] = ()   # gains between the conversion and the filter
    filt: Optional[Tuple[bool, int, float]] = None   # (high pass?, frequency, q)
    post: Tuple[float, ...] = ()  # gains behind the filter
    conv: bool = True


@dataclass
class Case:
    name: str
    ch: int
    mix_rate: int
    rows: List[Row]
    G: int                                   # rows per CTA the planner must choose
    launches: Tuple[str, ...]                # "default" and / or "chain"
    paths: Dict[str, Tuple[str, ...]]        # per launch: stage-A paths the batch is designed to take (count > 0)
    never: Dict[str, Tuple[str, ...]] = field(default_factory=dict)   # per launch: paths that must not run at all
    env: Dict[str, str] = field(default_factory=dict)                 # process environment of the default launch

    @property
    def starts(self):
        return [r.start for r in self.rows]

    def sources(self):
        out = []
        for r in self.rows:
            s = rb.TestSource(r.pcm, self.ch, r.rate)
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
            out.append(s)
        return out


# ------------------------------------------------------------------ planner and row-map mirrors (rb_fused.cu)
def reduced(frm, to):
    g = math.gcd(frm, to)
    return frm // g, to // g


def rows_per_cta(sms, S, ch, has_b, narrow):
    """G of rb_fused_try_create for a k_fused_hot batch; extends test_bench_geometries_gpu._hot_rows_per_cta with the wide stride
    and the filter-free plan.  narrow: mono rows that all interpolate with qT <= 238 (window + offset <= 244 floats): 32 rows;
    otherwise 28.  Filter-free batches of more than one stream per SM fill their CTAs and spread the timeline instead."""
    max_g = 32 if (narrow and ch == 1 and has_b) else 28
    k = -(-S // (sms * max_g))
    G = -(-S // (sms * k))
    if not has_b and S > sms:
        nx = -(-S // max_g)
        G = -(-S // nx)
    return max(1, min(G, max_g))


def q_tile(rate, mix_rate, ch):
    f, t = reduced(rate, mix_rate)
    return (TT // ch) * f // t


def is_narrow(rows, mix_rate, ch):
    return ch == 1 and all(r.conv and r.rate != mix_rate and 3 + q_tile(r.rate, mix_rate, 1) + 3 <= 244 for r in rows)


def row_pairs(G, chain):
    """(first, second) rows of the stage-A warps of a CTA with G rows (hot_first_row / hot_second_row)."""
    pairs = []
    for slot in range(23):
        first = slot if (chain or slot < 6) else (-1 if slot < 8 else slot - 2)
        j = slot if slot < 6 else {9: 6, 10: 7, 8: 8, 12: 9, 13: 10}.get(slot, -1)
        second = (23 if chain else 21) + j if j >= 0 else -1
        if 0 <= first < G and 0 <= second < min(G, 32):
            pairs.append((first, second))
    return pairs


def out_frames(L, rate, mix_rate, conv=True):
    """Frames UniformSourceIterator yields for L input frames (sample_rate.rs): frame n interpolates input frames
    (floor(n f / t), +1) while the right one exists; the first n whose left frame is the last one yields that frame alone."""
    f, t = reduced(rate, mix_rate)
    if not conv or f == t or L == 0:
        return L
    n = ((L - 1) * t + f - 1) // f
    return n + (1 if n * f // t == L - 1 else 0)


def out_len(r, case):
    return out_frames(r.pcm.size // case.ch, r.rate, case.mix_rate, r.conv) * case.ch


def row_tiles(case):
    """Row-tiles stage A walks: for every row, the tiles of the mixer timeline that overlap [start, start + out_len)."""
    total = 0
    for r in case.rows:
        n = out_len(r, case)
        if n:
            total += (r.start + n - 1) // TT - r.start // TT + 1
    return total


# ------------------------------------------------------------------ the float64 restatement
def lerp64(x, rate, mix_rate):
    f, t = reduced(rate, mix_rate)
    L = x.shape[0]
    if f == t or L == 0:
        return x
    n = np.arange(((L - 1) * t + f - 1) // f, dtype=np.int64)
    i0, num = n * f // t, n * f % t
    y = x[i0] + (x[i0 + 1] - x[i0]) * (num.astype(np.float64) / t)[:, None]
    if n.size * f // t == L - 1:
        y = np.concatenate([y, x[L - 1:L]])
    return y


def f64_stream(r, case):
    x = r.pcm.astype(np.float64).reshape(-1, case.ch)
    gain = lambda v: float(np.float32(v))
    for g in r.pre:
        x = x * gain(g)
    if r.conv:
        x = lerp64(x, r.rate, case.mix_rate)
    for g in r.mid:
        x = x * gain(g)
    if r.filt and x.shape[0]:
        high, f, q = r.filt
        b0, b1, b2, a1, a2 = (float(v) for v in oracle.blt_coeffs(high, f, q, case.mix_rate))
        x = scipy.signal.lfilter([b0, b1, b2], [1.0, a1, a2], x, axis=0)
    for g in r.post:
        x = x * gain(g)
    return x.reshape(-1)


def f64_mix(case):
    ys = [f64_stream(r, case) for r in case.rows]
    total = np.zeros(max(r.start + y.size for r, y in zip(case.rows, ys)), dtype=np.float64)
    for r, y in zip(case.rows, ys):
        total[r.start:r.start + y.size] += y
    return total


# ------------------------------------------------------------------ designed batches
def _gains(rng, n):
    return tuple(float(np.float32(0.4 + 1.2 * rng.random())) for _ in range(n))


def _filter(rng):
    return (bool(rng.random() < 0.3), int(rng.integers(150, 4000)), float(np.float32(0.4 + 0.8 * rng.random())))


def _frames_ending_at(start, rate, mix_rate, ch, residue, lo=1800):
    for L in range(lo, lo + 4 * TT):
        if (start + out_frames(L, rate, mix_rate) * ch) % TT == residue:
            return L
    raise AssertionError("no length ends there")


def designed(name, sms, S, rates, *, ch=1, mix_rate=48000, seed=0, n_pre=0, n_mid=0, n_post=1, filt=True, conv=True,
             specials=True, unsafe=False, launches=("default",), paths=None, never=None, env=None):
    """S rows, CTA after CTA.  In each CTA the first 21 rows start together and the rest start OFFSETS later (sorted), so that
    the warps' second rows meet their first rows at offsets that are multiples of every `to` (0, 480 for 147/160 and 2/3), of
    some (147, 160, 320, 441) or of none (37, 197, 517).  Rates are drawn per row; every row has its own filter and gains.
    specials: two rows per CTA of 0 or 1 frames, or ending exactly on / one frame past a tile boundary.
    unsafe: denormal differences, 3e30 and signed zeros in the first row only, the second row only or both rows of a pair, in
    the same tile of the mixer timeline."""
    rng = np.random.default_rng(seed)
    proto = [Row(np.zeros(0, np.float32), r, 0, conv=conv) for r in rates]
    G = rows_per_cta(sms, S, ch, filt, is_narrow(proto, mix_rate, ch))
    partner = {b: a for a, b in row_pairs(32, False)}
    rows = []
    for c in range(-(-S // G)):
        n = min(G, S - c * G)
        offs = [0] * min(n, 21) + sorted(int(v) for v in rng.choice(OFFSETS, max(0, n - 21)))
        special = {int(k): (c + j) % 4 for j, k in enumerate(rng.choice(n, 2, replace=False))} if specials and n > 1 else {}
        cta = []
        for g in range(n):
            rate = int(rng.choice(rates))
            if g in partner and rng.random() < 0.6:
                rate = cta[partner[g]].rate          # a second row mostly has its first row's rate
            start = ch * (c * CTA_SPAN + offs[g])
            L = int(rng.integers(1800, 2600))
            kind = special.get(g)
            if kind == 0:
                L = 0
            elif kind == 1:
                L = 1
            elif kind in (2, 3):
                L = _frames_ending_at(start, rate, mix_rate, ch, 0 if kind == 2 else ch) if conv else \
                    next(x for x in range(1800, 1800 + TT) if (start + x * ch) % TT == (0 if kind == 2 else ch))
            pcm = noise(L * ch, seed * 100003 + c * 97 + g)
            cta.append(Row(pcm, rate, start, _gains(rng, n_pre), _gains(rng, n_mid), _filter(rng) if filt else None,
                           _gains(rng, n_post), conv))
        if unsafe:
            _plant_unsafe(cta, c, ch, mix_rate)
        rows += cta
    assert [r.start for r in rows] == sorted(r.start for r in rows)
    default_paths = ("pair", "solo", "strided") if ch == 1 else ("solo", "strided")
    return Case(name, ch, mix_rate, rows, G, launches, paths or {l: default_paths for l in launches},
                {l: ("pair_failed", "redo") for l in launches} if never is None else never, env or {})


def _plant_unsafe(cta, c, ch, mix_rate):
    """Operands outside the exact-reciprocal range in the tile of the mixer timeline both rows of a pair cover: the first row
    only, the second only, or both (the pair vote fails, the rows run solo, the one with the bad operand redoes its tile)."""
    for p, (a, b) in enumerate(row_pairs(len(cta), False)):
        mode = (p + c) % 4
        if mode == 0:
            continue
        ra, rb_ = cta[a], cta[b]
        lo = max(ra.start, rb_.start)
        hi = min(ra.start + out_frames(ra.pcm.size, ra.rate, mix_rate) * ch, rb_.start + out_frames(rb_.pcm.size, rb_.rate, mix_rate) * ch)
        pos = (lo // TT + 2 + p % 3) * TT + 100
        if pos + 300 > hi:
            continue
        kind = (c + p) % 6
        for r, on in ((ra, mode in (1, 3)), (rb_, mode in (2, 3))):
            if not on:
                continue
            f, t = reduced(r.rate, mix_rate)
            i = (pos - r.start) // ch * f // t
            if kind == 0 and c % 4 == 0:
                vals = [3e30, -3e30, 1.0]
            elif kind == 1:
                vals = [0.0, -0.0, -0.0, 0.0, -0.0]
            else:
                vals = list(noise(6, c * 31 + p) * np.float32(1e-38))
            r.pcm[i:i + len(vals)] = np.asarray(vals, dtype=np.float32)


def _cases(sms):
    S32, S28 = 32 * sms, 28 * sms
    both = ("default", "chain")
    unsafe_paths = ("pair", "pair_failed", "solo", "redo", "strided")
    return {
        # 1. 32 mono rows per CTA, only gains behind the filter: stage A without gains (NOGAIN); one gain, then two (NPOST = -1)
        "mono32_post1": lambda: designed("mono32_post1", sms, S32, RATES_A, seed=1, launches=both),
        "mono32_post2": lambda: designed("mono32_post2", sms, S32, RATES_A, seed=2, n_post=2),
        # 2. gains in front of the conversion and between conversion and filter: hot_stage_a_pair<false, true>
        "mono32_front_gains": lambda: designed("mono32_front_gains", sms, S32, RATES_A, seed=3, n_pre=1, n_mid=1, launches=both),
        # 3. operands outside the guarded range in one or both rows of a pair
        "mono32_unsafe": lambda: designed("mono32_unsafe", sms, S32, (44100,), seed=4, specials=False, unsafe=True, launches=both,
                                          paths={"default": unsafe_paths, "chain": unsafe_paths}, never={}),
        # 4. the narrow stride at its limit: qT = 238 (241 taps) plus a window offset of up to 3 = 244 floats; with 44.9 kHz
        #    (qT = 239) rows the batch takes the wide stride and at most 28 rows
        "narrow_limit": lambda: designed("narrow_limit", sms, S32, (44700, 44800, 44700, 44800, 44100), seed=5),
        "wide_44k9_28": lambda: designed("wide_44k9_28", sms, S28, (44700, 44800, 44900), seed=6),
        # 5. a partial last CTA (25 rows), one second row per CTA, none
        "partial_last_cta": lambda: designed("partial_last_cta", sms, S32 - 7, RATES_A, seed=7),
        "rows22": lambda: designed("rows22", sms, 22 * sms, RATES_A, seed=8),
        "rows21": lambda: designed("rows21", sms, 21 * sms, RATES_A, seed=9, paths={"default": ("solo", "strided")},
                                   never={"default": ("pair", "pair_failed", "redo")}),
        # 6. 28-row wide CTAs: rates down and up, and rows without a conversion (strided path only)
        "wide_mixer_44k1": lambda: designed("wide_mixer_44k1", sms, S28, (48000, 48000, 32000), mix_rate=44100, seed=10),
        "wide_mixer_48k": lambda: designed("wide_mixer_48k", sms, S28, (52000, 44900, 44100), seed=11),
        "direct_48k": lambda: designed("direct_48k", sms, S28, (48000,), seed=12, conv=False, paths={"default": ("strided",)},
                                       never={"default": ("pair", "pair_failed", "solo", "redo")}),
        # 7. stereo, 28 rows, both recurrence warps: no pair pass
        "stereo28": lambda: designed("stereo28", sms, S28, RATES_A, ch=2, seed=13, launches=both,
                                     never={l: ("pair", "pair_failed", "redo") for l in both}),
        # 8. a 24-row chain (one second row per warp of the 23 + 9 map), the filter-free chain with per-row gains in front
        #    (k_fused_hot<1, false, true>: hot_stage_a_pair<false, false>); 9. the same batch in a default launch
        #    (k_fused_hot<1, false, false>) with the segment plan of the lane kernels switched off
        "chain24": lambda: designed("chain24", sms, 24 * sms, RATES_A, seed=14, launches=("chain",)),
        "filter_free28": lambda: designed("filter_free28", sms, S28, RATES_A, seed=15, n_pre=1, n_mid=1, n_post=0, filt=False,
                                          launches=both, env={"RB_SEGMENTS_FROM": str(1 << 40)}),
    }


CASE_NAMES = list(_cases(H100_SMS))


@functools.lru_cache(maxsize=2)
def build_case(name, sms):
    return _cases(sms)[name]()


@contextlib.contextmanager
def environ(values):
    old = {k: os.environ.get(k) for k in values}
    os.environ.update(values)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def render(ctx, case, launch, debug_lib=None):
    """Mixer output of one launch (rendered twice: the second must repeat the first); with debug_lib, also the stage-A path
    counters of the render."""
    flags = capi.RB_MIX_EXACT_ORDER if launch == "chain" else 0
    counts = None
    with environ(case.env if launch == "default" else {}):
        with rb.Batch(case.sources(), case.ch, case.mix_rate, flags=flags, mix_starts=case.starts, ctx=ctx) as b:
            assert b.kernel_family == 1, f"{case.name}: kernel family {b.kernel_family}"
            group = b.mix_group
            b.upload_all()
            if debug_lib is not None:
                import ctypes
                buf = (ctypes.c_ulonglong * 8)()
                assert debug_lib.rb_debug_hot_paths(buf, 1) == 0
            got = b.render_mix()
            if debug_lib is not None:
                assert debug_lib.rb_debug_hot_paths(buf, 0) == 0
                counts = dict(zip(PATHS, list(buf)))
            again = b.render_mix()
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32)), f"{case.name} {launch}: render is not idempotent"
    return got, group, counts


def _paths_child():
    """Runs in a process of its own on the instrumented library (RODIO_B200_LIB): every case and launch, one render each;
    prints the counters as JSON."""
    import ctypes
    ctx = rb.default_context(0)
    lib = ctypes.CDLL(os.environ["RODIO_B200_LIB"])
    lib.rb_debug_hot_paths.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    out = {}
    for name in CASE_NAMES:
        case = build_case(name, ctx.sm_count)
        for launch in case.launches:
            out[f"{name}:{launch}"] = render(ctx, case, launch, lib)[2]
    print(json.dumps(out))


# ------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_hot_rows(ctx, name):
    case = build_case(name, ctx.sm_count)
    srcs = case.sources()
    per_stream = [oracle.chain_uniform(to_oracle(s), case.ch, case.mix_rate) for s in srcs]
    ref = oracle.mixer([to_oracle(s, st) for s, st in zip(srcs, case.starts)], case.ch, case.mix_rate)
    truth = f64_mix(case)
    assert truth.size == ref.size
    peak = float(np.max(np.abs(truth)))
    e_ref = float(np.max(np.abs(ref - truth)))
    for launch in case.launches:
        got, group, _ = render(ctx, case, launch)
        if launch == "chain":
            assert group == 0
            assert_bit_exact(got, ref, f"{name}, exact-order chain vs the reference's sequential mixer")
        else:
            assert group == case.G, f"{name}: {group} rows per CTA, expected {case.G}"
            want = grouped_expected_mix(per_stream, case.starts, ref.size, case.G)
            assert_bit_exact(got, want, f"{name}, default launch vs oracle streams added in the kernel's order")
        e_got = float(np.max(np.abs(got - truth)))
        assert e_got <= F64_FACTOR * e_ref + 1e-7 * peak, f"{name} {launch}: {e_got:.3e} from the f64 chain, reference {e_ref:.3e}"


@pytest.fixture(scope="session")
def hot_paths(built, tmp_path_factory):
    """Stage-A path counters of every case and launch, from an instrumented build of the library (-DRB_HOT_PATHS) run in a
    process of its own."""
    from rodio_b200 import build as rb_build
    lib = rb_build.build(force=True, extra_flags=["-DRB_HOT_PATHS"],
                         out=str(tmp_path_factory.mktemp("hot_paths") / "librodio_b200_paths.so"))
    env = dict(os.environ, RODIO_B200_LIB=lib)
    env.pop("RB_SEGMENTS_FROM", None)
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; "
            f"import test_hot_rows_gpu as t; t._paths_child()")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_stage_a_paths(ctx, hot_paths, name):
    """Every path the case was designed for ran, the ones it must not take did not, and stage A walked exactly the row-tiles the
    rows cover (a pair counts two; a failed pair vote is counted again on the solo path)."""
    case = build_case(name, ctx.sm_count)
    for launch in case.launches:
        n = hot_paths[f"{name}:{launch}"]
        print(f"\n{name} {launch} {n}")
        for p in case.paths[launch]:
            assert n[p] > 0, f"{name} {launch}: no row-tile took the {p} path: {n}"
        for p in case.never.get(launch, ()):
            assert n[p] == 0, f"{name} {launch}: {n[p]} row-tiles took the {p} path: {n}"
        walked = n["pair"] + n["solo"] + n["redo"] + n["strided"]
        assert walked == row_tiles(case), f"{name} {launch}: stage A walked {walked} row-tiles, the rows cover {row_tiles(case)}"


@pytest.mark.gpu
def test_one_44k9_row_takes_the_wide_stride(ctx):
    """One 44.9 kHz row (qT = 239: 242 taps + offset > 244 floats) in the 32-row batch of test_hot_rows[narrow_limit]: the planner
    falls back to the wide stride and at most 28 rows per CTA."""
    case = build_case("narrow_limit", ctx.sm_count)
    srcs = case.sources()
    srcs[5] = rb.UniformSourceIterator(rb.TestSource(case.rows[5].pcm, 1, 44900), 1, 48000).low_pass(1000).amplify(0.9)
    rows = list(case.rows)
    rows[5] = Row(case.rows[5].pcm, 44900, case.rows[5].start)
    assert not is_narrow(rows, 48000, 1) and is_narrow(case.rows, 48000, 1)
    with rb.Batch(srcs, 1, 48000, mix_starts=case.starts, ctx=ctx) as b:
        assert b.kernel_family == 1
        assert b.mix_group == rows_per_cta(ctx.sm_count, len(srcs), 1, True, False) != case.G


# ------------------------------------------------------------------ CPU: the reference, the designs, the planner arithmetic
@pytest.mark.parametrize("name", CASE_NAMES)
def test_f64_reference_matches_oracle(name):
    """The float64 restatement agrees with the oracle on every designed batch: the same length for every stream and for the mix,
    within 1e-5 of the peak; and the oracle's streams added in the kernel's order stay within the bound test_hot_rows applies."""
    case = build_case(name, H100_SMS)
    srcs = case.sources()
    per_stream = [oracle.chain_uniform(to_oracle(s), case.ch, case.mix_rate) for s in srcs]
    for r, y in zip(case.rows, per_stream):
        assert y.size == out_len(r, case)
        if y.size:
            e = float(np.max(np.abs(y - f64_stream(r, case))))
            assert e <= 1e-4 * float(np.max(np.abs(y))) + 1e-30, (r.rate, r.filt, e)
    ref =oracle.mixer([to_oracle(s, st) for s, st in zip(srcs, case.starts)], case.ch, case.mix_rate)
    truth = f64_mix(case)
    assert truth.size == ref.size
    peak = float(np.max(np.abs(truth)))
    e_ref = float(np.max(np.abs(ref - truth)))
    assert e_ref <= 1e-4 * peak, (e_ref, peak)
    if "default" in case.launches:
        grouped = grouped_expected_mix(per_stream, case.starts, ref.size, case.G)
        e_grouped = float(np.max(np.abs(grouped - truth)))
        assert e_grouped <= 1.5 * e_ref + 1e-7 * peak, (e_grouped, e_ref, peak)


def _pair_kinds(case, chain):
    """How the two rows of each warp relate, counted over the batch."""
    kinds = dict.fromkeys(("equal", "offset", "other_r0", "other_rate", "ragged"), 0)
    G = case.G
    for c0 in range(0, len(case.rows), G):
        cta = case.rows[c0:c0 + G]
        for a, b in row_pairs(len(cta), chain):
            ra, rb_ = cta[a], cta[b]
            if ra.rate != rb_.rate:
                kinds["other_rate"] += 1
                continue
            d = (rb_.start - ra.start) // case.ch
            to = reduced(ra.rate, case.mix_rate)[1]
            kinds["equal" if d == 0 else "offset" if d % to == 0 else "other_r0"] += 1
            if d % to == 0 and ra.start + out_len(ra, case) != rb_.start + out_len(rb_, case):
                kinds["ragged"] += 1
    return kinds


@pytest.mark.parametrize("name", ["mono32_post1", "mono32_front_gains", "partial_last_cta", "narrow_limit", "chain24"])
def test_designs_pair_rows_every_way(name):
    """The designed batches put first and second rows together in every relation under the row map of each launch, and hold
    rows of 0 and 1 frames and rows that end on and one frame past a tile boundary."""
    case = build_case(name, H100_SMS)
    for launch in case.launches:
        kinds = _pair_kinds(case, launch == "chain")
        assert min(kinds.values()) >= 3, (launch, kinds)
    ends = [(r.start + out_len(r, case)) % TT for r in case.rows if r.pcm.size > 1]
    sizes = [r.pcm.size for r in case.rows]
    assert 0 in sizes and 1 in sizes and 0 in ends and 1 in ends


def test_narrow_window_fits_its_stride():
    """The bulk copy of a row's input window (hot_issue_window: woff + min(qT + 3, frames left) frames, rounded up to 16 bytes)
    never passes the row's stride: 244 floats when every row has qT <= 238 (32 rows per CTA), 320 otherwise.  The narrow-limit
    batch fills the 244 floats exactly (qT = 238, woff = 3) and the wide one would not fit them."""
    for qT in range(0, 239):
        for woff in range(4):
            assert ((woff + qT + 3) * 4 + 15) // 16 * 16 <= 244 * 4
    for ch, stride in ((1, 320), (2, 320)):
        for qT in range(0, 400):
            if 3 + (qT + 3) * ch <= stride:       # the planner's window_fits
                woff_max = 3 if ch == 1 else 2    # (i0 * C) & 3
                assert ((woff_max + (qT + 3) * ch) * 4 + 15) // 16 * 16 <= stride * 4
    assert q_tile(44700, 48000, 1) == q_tile(44800, 48000, 1) == 238 and q_tile(44900, 48000, 1) == 239
    case = build_case("narrow_limit", H100_SMS)
    assert case.G == 32 and is_narrow(case.rows, 48000, 1)
    most = 0
    for r in case.rows:
        f, t = reduced(r.rate, 48000)
        L, n, qT = r.pcm.size, out_len(r, case), q_tile(r.rate, 48000, 1)
        for m0 in range(r.start // TT * TT, r.start + n, TT):
            i0 = (max(m0, r.start) - r.start) * f // t
            floats = (i0 & 3) + min(qT + 3, L - i0)
            assert floats <= 244
            most = max(most, floats)
    assert most == 244
    assert not is_narrow(build_case("wide_44k9_28", H100_SMS).rows, 48000, 1)
