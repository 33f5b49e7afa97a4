"""k_lerp_mix (kernel family 6) on batches whose rows differ.

Family 6 serves every filter-free mono batch (resample -> [one gain] -> mix) of 64 to 1023 in-phase streams, and with
RB_MIX_EXACT_ORDER such batches of any size below 1024 streams, in one group.  A CTA owns one tile of 1024 timeline frames and
one group of rows; it derives the tile's first input frame (i_tile) and the window width (n_win) from the batch's origin (the
earliest start of a non-empty stream), sends a row through a shared-memory window when the row interpolates on the whole tile
and its inputs are inside the exact-reciprocal class, and through global memory with the IEEE division otherwise.  The
designs below put each of these choices at every position of a 4-row stage, in groups of every shape, at timeline ends,
origins inside and on tile boundaries, every window alignment, seven rate pairs, special inputs and gains.

Every design is checked on the device
  * for the kernel and launch the planner's rule gives (rb_lanes_batch.cu): family 6, the rows per group, one launch for one
    group and two otherwise;
  * bit for bit against the oracle's per-stream outputs added in the kernel's documented order (per group from +0.0 in the
    planner's stream order, the group partials in group order), and in exact order against the reference's sequential mixer
    (NaN only has to meet NaN; payloads are not compared);
  * the same on a second render, and after inputs are uploaded again;
  * within twice the oracle's own distance of a float64 restatement.
The CPU tests pin the float64 restatement against the oracle, restate the kernel's tile arithmetic with 64-bit wrap-around to
show that every design reaches the paths it claims and reads only inside its rows' inputs, and run the designs on the
host-emulated library, whose k_lerp_mix follows the kernel and checks every read."""
import functools
import os
import subprocess
import sys
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import pytest

import oracle
import rodio_b200 as rb
from helpers import assert_close_peak, noise, to_oracle
from rodio_b200 import capi
from test_bench_geometries_gpu import grouped_expected_mix
from test_generic_fused_rows_gpu import assert_same_mix, f64_distance
from test_hot_rows_gpu import F64_FACTOR, H100_SMS, lerp64, out_frames, reduced

TILE = 1024                     # timeline frames per CTA (256 threads x LM_U)
LM_ROWS, LM_GROUP, LM_WQ = 4, 64, 260   # rows per stage, row descriptors staged at a time, 16-byte quads of a window
M64 = (1 << 64) - 1
SPECIALS = (1e-41, 2.0 ** 61, np.inf, -np.inf, np.nan)   # outside the exact-reciprocal class ([2^-70, 2^60] and 0)


@dataclass
class Row:
    pcm: np.ndarray             # mono f32
    start: int                  # mixer frames
    gain: float = 1.0           # the one gain behind the conversion (used when the case has gains)
    span: int = 0               # span_len the source reports (0: none, like TestSource)


@dataclass
class Case:
    name: str
    rate: int
    mix_rate: int
    rows: List[Row]             # in the order they are handed to the mixer
    exact: bool = False
    gains: bool = True
    claims: tuple = ()          # paths and shapes the design must reach (see walk())
    uploads: List[Dict[int, np.ndarray]] = field(default_factory=list)   # inputs rewritten between renders (stream index -> pcm)
    family: Optional[int] = 6   # planner edges: the family the batch must take (None: anything but 6)

    @property
    def flags(self):
        return capi.RB_MIX_EXACT_ORDER if self.exact else 0

    @functools.cached_property
    def order(self):
        """The planner's stream order: a stable sort by start."""
        return sorted(range(len(self.rows)), key=lambda i: self.rows[i].start)

    def source(self, r, pcm=None):
        s = rb.Source(r.pcm if pcm is None else pcm, 1, self.rate, span_len=r.span)
        s = rb.UniformSourceIterator(s, 1, self.mix_rate)
        return s.amplify(r.gain) if self.gains else s

    def sources(self):
        return [self.source(r) for r in self.rows]


# ------------------------------------------------------------------ planner mirror (rb_lanes_batch.cu)
def plan_groups(case, sms):
    """(groups, rows per group) of the k_lerp_mix plan: about two waves of CTAs, at most 64 and at least 16 rows per group."""
    n = len(case.rows)
    if case.exact:
        return 1, n
    mix_len = mix_length(case, [r.pcm for r in case.rows])
    tiles = -(-mix_len // TILE)
    groups = max(-(-2 * sms // tiles), -(-n // 64))
    groups = max(1, min(groups, -(-n // 16)))
    per = -(-n // groups)
    return -(-n // per), per


def mix_length(case, pcms):
    return max(r.start + out_frames(p.size, case.rate, case.mix_rate) for r, p in zip(case.rows, pcms))


def in_class(p):
    a = np.abs(p.astype(np.float64))
    return bool(np.all((a == 0) | ((a >= 2.0 ** -70) & (a < 2.0 ** 60))))


def signed64(v):
    v &= M64
    return v - (1 << 64) if v >> 63 else v


def walk(case, sms, pcms=None, parent=False):
    """The kernel's tile arithmetic over every (group, tile, row), restated with 64-bit wrap-around (parent: the parent commit's
    i_tile = (tile_lo - origin) * from / to).  Returns the paths taken and every read outside a row's input, which is the row's
    frames rounded out to 16-byte granules (inputs are 16-byte aligned)."""
    pcms = [r.pcm for r in case.rows] if pcms is None else pcms
    f, t = reduced(case.rate, case.mix_rate)
    rows = []
    for i in case.order:
        L, s = pcms[i].size, case.rows[i].start
        n = out_frames(L, case.rate, case.mix_rate)
        n_int = min(((L - 1) * t + f - 1) // f, n) if L >= 2 else 0
        rows.append(dict(L=L, lo=s, hi_int=s + n_int, hi=s + n, empty=n == 0, unsafe=not in_class(pcms[i])))
    origin = min(r["lo"] for r in rows if not r["empty"])
    for r in rows:
        r["shift"] = 0 if r["empty"] else (r["lo"] - origin) // t * f
    mix_len = mix_length(case, pcms)
    groups, per = plan_groups(case, sms)
    st = dict(window=0, glob=0, offs=set(), win_pos=set(), glob_pos=set(), unsafe_pos=set(), origin_inside=False, silent_group_tile=False,
              chunks=False, partial_window=False, raw_tail_last_tile=False, max_n_win=0, bad=[])
    last_lo = (mix_len - 1) // TILE * TILE
    for r in rows:
        if not r["empty"] and r["hi_int"] < r["hi"] and r["hi"] > last_lo:
            st["raw_tail_last_tile"] = True
    for g in range(groups):
        r_lo, r_hi = g * per, min(len(rows), (g + 1) * per)
        st["chunks"] |= r_hi - r_lo > LM_GROUP
        for tile_lo in range(0, mix_len, TILE):
            tile_hi = min(mix_len, tile_lo + TILE)
            base = tile_lo if parent else max(tile_lo, origin)
            i_tile = (((base - origin) & M64) * f & M64) // t
            n_win = ((((((max(tile_hi - 1, base) - origin) & M64) * f & M64) // t - i_tile) & 0xffffffff) + 2) & 0xffffffff
            if tile_lo < origin < tile_hi:
                st["origin_inside"] = True
            win_ok = n_win + 3 <= LM_WQ * 4
            active = False
            for k in range(r_lo, r_hi):
                r = rows[k]
                stage_pos = ((k - r_lo) % LM_GROUP) % LM_ROWS
                rel = signed64(i_tile - r["shift"])           # float offset of row.p + i_tile from the row's input
                granules = -(-r["L"] // 4) * 4
                if win_ok and not r["unsafe"] and r["lo"] <= tile_lo and r["hi_int"] >= tile_hi:
                    off = rel & 3
                    nq = (off + n_win + 3) >> 2
                    st["window"] += 1
                    st["offs"].add(off)
                    st["win_pos"].add(stage_pos)
                    st["max_n_win"] = max(st["max_n_win"], n_win)
                    st["partial_window"] |= tile_hi - tile_lo < TILE
                    active = True
                    if rel - off < 0 or rel - off + 4 * nq > granules:
                        st["bad"].append((g, tile_lo, k, "window", rel - off, rel - off + 4 * nq, r["L"]))
                    continue
                n = np.arange(max(r["lo"], tile_lo), min(r["hi"], tile_hi), dtype=np.int64)
                if r["hi"] <= tile_lo or r["lo"] >= tile_hi or n.size == 0:    # silent here (an empty row reads nothing)
                    continue
                active = True
                st["glob"] += 1
                st["glob_pos"].add(stage_pos)
                if r["unsafe"]:
                    st["unsafe_pos"].add(stage_pos)
                i = (np.maximum(n, base) - origin) * f // t if not parent else (n - origin) * f // t
                tap = (i - (i_tile & 0xffffffff)) & 0xffffffff
                reads = [signed64(i_tile + int(tap.min()) - r["shift"]), signed64(i_tile + int(tap.max()) - r["shift"])]
                if (n < r["hi_int"]).any():
                    reads.append(signed64(i_tile + int(tap[n < r["hi_int"]].max()) + 1 - r["shift"]))
                if min(reads) < 0 or max(reads) >= granules:
                    st["bad"].append((g, tile_lo, k, "global", min(reads), max(reads), r["L"]))
            st["silent_group_tile"] |= groups > 1 and not active
    return st


# ------------------------------------------------------------------ the float64 restatement
def f64_mix(case, pcms):
    w = lambda r: float(np.float32(r.gain)) if case.gains else 1.0
    ys = [lerp64(p.astype(np.float64).reshape(-1, 1), case.rate, case.mix_rate).reshape(-1) * w(r) for r, p in zip(case.rows, pcms)]
    total = np.zeros(mix_length(case, pcms), dtype=np.float64)
    with np.errstate(all="ignore"):
        for r, y in zip(case.rows, ys):
            total[r.start:r.start + y.size] += y
    return total


def expected(case, pcms, sms):
    """The kernel's documented order (or the reference's sequential mixer in exact order), the reference, the f64 restatement."""
    srcs = [case.source(r, p) for r, p in zip(case.rows, pcms)]
    ref = oracle.mixer([to_oracle(s, r.start) for s, r in zip(srcs, case.rows)], 1, case.mix_rate)
    if case.exact:
        return ref, ref, f64_mix(case, pcms)
    per = [oracle.chain_uniform(to_oracle(srcs[i]), 1, case.mix_rate) for i in case.order]
    groups, G = plan_groups(case, sms)
    want = grouped_expected_mix(per, [case.rows[i].start for i in case.order], ref.size, G)
    return want, ref, f64_mix(case, pcms)


# ------------------------------------------------------------------ designs
def _pcm(L, seed, amp=1.0):
    return noise(L, seed, amp)


def _ending_at(end, rate, origin=0, k0=0):
    """(start, input frames) of a row that starts at origin + k * to, k >= k0, and ends at timeline frame `end`."""
    f, t = reduced(rate, 48000)
    for k in range(k0, k0 + 16):
        out = end - origin - t * k
        for L in range(max(1, out * f // t - 3), out * f // t + 4):
            if out_frames(L, rate, 48000) == out:
                return origin + t * k, L
    return None


def _origin(o, exact, rate=44100, n=70, seed=0, empty_front=False, single=False):
    f, t = reduced(rate, 48000)
    rng = np.random.default_rng(seed + o)
    lens = (1, 2, 3, 40, 700, 1500, 3000, 4500)
    rows = [Row(_pcm(4000, seed + o), o, 0.75)]
    if not single:
        for k in range(1, n):
            rows.append(Row(_pcm(lens[k % 8], seed + o + k), o + t * int(rng.integers(0, 6)), 0.5 + 0.01 * k))
    if empty_front:
        rows.insert(0, Row(np.zeros(0, np.float32), 0, 2.0))
    claims = ("origin_inside",) if o % TILE else ()
    name = f"origin_{o}" + (f"_{rate}" if rate != 44100 else "") + ("_empty_front" if empty_front else "") + \
        ("_single" if single else "") + ("_exact" if exact else "")
    return Case(name, rate, 48000, rows, exact=exact, claims=claims)


def _stages(exact):
    """Window rows (long, from frame 0) and global rows (short) at every stage position, and late long rows whose shifts
    k * 147 give every window offset."""
    rows = []
    for i in range(48):
        long_ = ((i // 4) + i) % 2 == 0
        rows.append(Row(_pcm(6000 if long_ else 100 + 37 * i, 100 + i), 0, 0.9 - 0.01 * i))
    for k in range(24):
        rows.append(Row(_pcm(5200 - 40 * k, 200 + k), 160 * (1 + k % 8), 1.1 + 0.01 * k))
    return Case("stages" + ("_exact" if exact else ""), 44100, 48000, rows, exact=exact,
                claims=("win_pos_all", "glob_pos_all", "offs_all"))


def _reciprocal(exact):
    """Rows with inputs outside the exact-reciprocal class at every stage position beside safe rows (some with -0); a safe
    stream turned unsafe and an unsafe one turned safe by a new upload, then back."""
    rows = []
    for i in range(68):
        p = _pcm(4000, 300 + i)
        if i % 3 == 1 and i < 60:
            j = (i // 3) % len(SPECIALS)
            p[500 + 17 * i:503 + 17 * i] = np.float32(SPECIALS[j])
        if i % 5 == 0:
            p[100:140] = np.float32(-0.0)
            p[900:905] = np.float32(0.0)
        rows.append(Row(p, 0, 1.0 - 0.013 * i))
    unsafe0, safe0 = rows[1].pcm, rows[0].pcm
    to_unsafe = safe0.copy()
    to_unsafe[2000] = np.float32(2.0 ** 61)
    to_safe = _pcm(4000, 399)
    uploads = [{0: to_unsafe, 1: to_safe}, {0: safe0, 1: unsafe0}]
    return Case("reciprocal_class" + ("_exact" if exact else ""), 44100, 48000, rows, exact=exact, uploads=uploads,
                claims=("win_pos_all", "unsafe_pos_all"))


def _groups():
    """67 rows: 5 groups of 14 (not a multiple of 4) and a short last group of 11; the first group's rows end in tile 0, so
    that group is silent on every later tile (its partial row must stay +0 there)."""
    rows = [Row(_pcm(200 + 50 * i, 400 + i), 0, 0.8) for i in range(14)]
    rows += [Row(_pcm(3000, 420 + i), 160 * (10 + i % 30), 0.6 + 0.005 * i) for i in range(53)]
    return Case("groups_short_last_silent", 44100, 48000, rows, claims=("silent_group_tile",))


def _exact_chunks(n):
    rng = np.random.default_rng(500 + n)
    rows = []
    for i in range(n):
        L = int(rng.integers(1, 2500)) if i % 7 else 2500
        p = _pcm(L, 600 + i)
        if i % 11 == 3 and L > 10:
            p[L // 2] = np.float32(1e-40)
        rows.append(Row(p, 160 * int(rng.integers(0, 8)), 0.5 + 0.001 * i))
    return Case(f"exact_{n}_rows", 44100, 48000, rows, exact=True, claims=("chunks",) if n > LM_GROUP else ())


def _ends(mix_len, exact):
    """A timeline of exactly mix_len frames: window rows from the origin up to its last full tile, rows whose raw last frame lies
    inside the last tile, inputs of 0 .. 3 frames, ragged rows in between.  (A converted row always ends on one raw frame:
    hi_int = hi - 1, so no row interpolates on a partial last tile and the window path never takes one.)  44.1 -> 48 kHz never
    yields 63 frames modulo 160, so the origin moves where the end needs it."""
    rate = 44100
    o = next(o for o in range(160) if _ending_at(mix_len, rate, o))
    rows = []
    for k in range(4):
        s, L = _ending_at(mix_len - 5 * k, rate, o, k0=k) or _ending_at(mix_len - 5 * k - 1, rate, o, k0=k)
        rows.append(Row(_pcm(L, 700 + mix_len + k), s, 0.9 + 0.1 * k))
    for L in (0, 1, 2, 3, 0, 1, 2, 3):
        rows.append(Row(_pcm(L, 720 + L), o + 160 * (L + 1) if mix_len > 1023 else o + 160 * L, 0.7))
    rng = np.random.default_rng(mix_len)
    while len(rows) < 66:
        s = o + 160 * int(rng.integers(0, max(1, (mix_len - o - 200) // 160)))
        L = int(rng.integers(1, max(2, (mix_len - s) * 147 // 160 - 2)))
        rows.append(Row(_pcm(L, 730 + len(rows)), s, 0.4 + 0.01 * len(rows)))
    return Case(f"ends_{mix_len}" + ("_exact" if exact else ""), rate, 48000, rows, exact=exact,
                claims=("raw_tail_last_tile",) + (("origin_inside",) if o else ()))


def _ratio(rate, mix_rate, gains, n=66, L_max=3000):
    f, t = reduced(rate, mix_rate)
    rng = np.random.default_rng(rate + mix_rate)
    late = t <= 1280
    rows = []
    for i in range(n):
        s = t * int(rng.integers(0, 4)) if late and i else 0
        L = L_max if i % 4 == 0 else int(rng.integers(1, L_max))
        rows.append(Row(_pcm(L, 800 + i), s, 0.3 + 0.02 * i))
    claims = ("wide_window",) if (f, t) == (47999, 48000) else ()
    return Case(f"ratio_{rate}_{mix_rate}" + ("" if gains else "_no_gain"), rate, mix_rate, rows, gains=gains, claims=claims)


def _gain_values():
    """Per-row gains, 0, negative gains, and gains that overflow to +-Inf on window rows."""
    gains = (0.0, -0.5, 1.5, -3.0, 1e21, -1e21, 0.25, 2.0)
    rows = []
    for i in range(66):
        p = _pcm(3500 if i % 3 else 900, 900 + i)
        if abs(gains[i % 8]) == 1e21:                # inside the class: 1e18 * 1e21 overflows, 1e-16 * 1e21 stays audio-sized
            p *= np.float32(1e-16)
            p[600:700] = np.float32(1e18) * np.sign(p[600:700])
        rows.append(Row(p, 160 * (i % 5), gains[i % 8] * (1 + 0.01 * i) if gains[i % 8] else 0.0))
    return Case("gains", 44100, 48000, rows, claims=("win_pos_all",))


def _cases():
    c = []
    for o in (160, 480, 960, 1120, 2080, 5120):
        for exact in (False, True):
            c.append(_origin(o, exact, empty_front=o in (480, 2080)))
    c += [_origin(160, True, single=True), _origin(480, True, single=True)]
    c += [_origin(320, exact, rate=22050) for exact in (False, True)]
    c += [_stages(False), _stages(True), _reciprocal(False), _reciprocal(True), _groups()]
    c += [_exact_chunks(n) for n in (64, 65, 128, 129, 900)]
    c += [_ends(m, exact) for m in (1023, 2048, 2049) for exact in (False, True)]
    c += [_ratio(22050, 48000, False), _ratio(8000, 48000, True), _ratio(47999, 48000, True, L_max=2500), _ratio(32000, 44100, False),
          _ratio(11025, 96000, True, L_max=600), _ratio(44100, 48001, True)]
    c += [_gain_values()]
    return {x.name: x for x in c}


def _edges():
    """Batches next to family 6 that the planner must route elsewhere (or, for the smaller twin, keep)."""
    def plain(name, n, L, exact=False, family=6, rates=None, starts=None, span=False):
        rows = [Row(_pcm(L, 1000 + i), starts[i] if starts else 0, 0.9, span=L if span else 0) for i in range(n)]
        c = Case(name, 44100, 48000, rows, exact=exact, family=family)
        c.rates = rates or [44100] * n
        return c
    e = [plain("edge_1023_default", 1023, 600), plain("edge_1024_default", 1024, 4000, family=4),
         plain("edge_1023_exact", 1023, 600, exact=True), plain("edge_1024_exact", 1024, 600, exact=True, family=1),
         plain("edge_out_of_phase", 70, 2000, family=None, starts=[160 * (i % 4) + (37 if i == 33 else 0) for i in range(70)]),
         plain("edge_second_rate_pair", 70, 2000, family=None, rates=[44100] * 69 + [32000]),
         plain("edge_clip_32767", 64, 32767, span=True), plain("edge_clip_32768", 64, 32768, span=True),
         plain("edge_clip_32769", 64, 32769, span=True, family=None)]
    return {x.name: x for x in e}


CASES = _cases()
CASE_NAMES = list(CASES)
EDGES = _edges()
EDGE_NAMES = list(EDGES)


# ------------------------------------------------------------------ GPU tests
def _check(case, got, pcms, sms, what):
    want, ref, truth = expected(case, pcms, sms)
    if case.exact:
        assert_same_mix(got, ref, f"{what}: exact order vs the reference's sequential mixer")
    else:
        assert_same_mix(got, want, f"{what}: oracle streams added in the kernel's order")
    with np.errstate(all="ignore"):
        e_got, peak = f64_distance(got.astype(np.float64), truth)
        e_ref, _ = f64_distance(ref.astype(np.float64), truth)
    assert e_got <= F64_FACTOR * e_ref + 1e-7 * peak, f"{what}: {e_got:.3e} from the f64 restatement, reference {e_ref:.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_lerp_mix_rows(ctx, name):
    case = CASES[name]
    groups, per = plan_groups(case, ctx.sm_count)
    pcms = [r.pcm for r in case.rows]
    with rb.Batch(case.sources(), 1, case.mix_rate, flags=case.flags, mix_starts=[r.start for r in case.rows], ctx=ctx) as b:
        assert b.kernel_family == 6, f"{name}: kernel family {b.kernel_family}"
        assert b.mix_group == (per if groups > 1 else 0), f"{name}: {b.mix_group} rows per group, expected {per} in {groups}"
        assert b.launches_per_render == (2 if groups > 1 else 1)
        b.upload_all()
        for step in [{}] + case.uploads:
            for i, p in step.items():
                b.upload(i, p)
                pcms[i] = p
            got = b.render_mix()
            again = b.render_mix()
            assert np.array_equal(got.view(np.uint32), again.view(np.uint32)), f"{name}: the second render differs"
            _check(case, got, pcms, ctx.sm_count, f"{name} after {len(step)} re-uploads" if step else name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", EDGE_NAMES)
def test_planner_edges(ctx, name):
    case = EDGES[name]
    srcs = [rb.UniformSourceIterator(rb.Source(r.pcm, 1, rt, span_len=r.span), 1, 48000).amplify(r.gain) for r, rt in zip(case.rows, case.rates)]
    starts = [r.start for r in case.rows]
    ref = oracle.mixer([to_oracle(s, st) for s, st in zip(srcs, starts)], 1, 48000)
    with rb.Batch(srcs, 1, 48000, flags=case.flags, mix_starts=starts, ctx=ctx) as b:
        fam = b.kernel_family
        assert fam == case.family if case.family is not None else fam != 6, f"{name}: kernel family {fam}"
        b.upload_all()
        got = b.render_mix()
    if case.exact:
        assert_same_mix(got, ref, f"{name}: exact order")
    else:
        assert_close_peak(got, ref, 1e-5, f"{name}: family {fam} vs the sequential mixer")


# ------------------------------------------------------------------ CPU: the reference, the designs, the emulator
@pytest.mark.parametrize("name", CASE_NAMES)
def test_f64_reference_matches_oracle(name):
    """The float64 restatement agrees with the oracle: the same length for every stream and the mix, within 1e-5 of the peak
    where both are audio-sized; the oracle's streams added in the kernel's order stay within the bound test_lerp_mix_rows applies."""
    case = CASES[name]
    for r in case.rows:
        y = oracle.chain_uniform(to_oracle(case.source(r)), 1, case.mix_rate)
        assert y.size == out_frames(r.pcm.size, case.rate, case.mix_rate)
    pcms = [r.pcm for r in case.rows]
    want, ref, truth = expected(case, pcms, H100_SMS)
    assert ref.size == truth.size == want.size
    with np.errstate(all="ignore"):
        e_ref, peak = f64_distance(ref.astype(np.float64), truth)
        e_want, _ = f64_distance(want.astype(np.float64), truth)
    assert peak > 0 and e_ref <= 1e-5 * peak, (e_ref, peak)
    assert e_want <= F64_FACTOR * e_ref + 1e-7 * peak, (e_want, e_ref, peak)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_designs_reach_their_paths_and_stay_inside_their_inputs(name):
    """The kernel's tile arithmetic, restated with 64-bit wrap-around: every design takes the paths it claims, reads only inside
    its rows' inputs -- and an origin inside a tile made the parent commit's formula read far outside them."""
    case = CASES[name]
    for pcms in [[r.pcm for r in case.rows]] + [[step.get(i, r.pcm) for i, r in enumerate(case.rows)] for step in case.uploads]:
        st = walk(case, H100_SMS, pcms)
        assert not st["bad"], f"{name}: reads outside a row's input: {st['bad'][:3]}"
        claims = {"origin_inside": st["origin_inside"], "win_pos_all": st["win_pos"] == {0, 1, 2, 3},
                  "glob_pos_all": st["glob_pos"] == {0, 1, 2, 3}, "offs_all": st["offs"] == {0, 1, 2, 3},
                  "unsafe_pos_all": st["unsafe_pos"] == {0, 1, 2, 3}, "silent_group_tile": st["silent_group_tile"],
                  "chunks": st["chunks"], "partial_window": st["partial_window"], "raw_tail_last_tile": st["raw_tail_last_tile"],
                  "wide_window": st["max_n_win"] == 1025}
        for c in case.claims:
            assert claims[c], f"{name}: does not reach {c}: {st}"
    parent = walk(case, H100_SMS, parent=True)
    if "origin_inside" in case.claims:
        assert parent["bad"] and all(b[1] < min(r.start for r in case.rows if r.pcm.size) for b in parent["bad"]), parent["bad"][:3]
    else:
        assert not parent["bad"]


def test_planner_edges_are_what_they_claim():
    """The edge batches sit where the planner's rules put them: stream counts around 1024, one stream out of phase, a second
    rate pair, span restarts from 32 769 samples on."""
    assert [len(EDGES[n].rows) for n in ("edge_1023_default", "edge_1024_default", "edge_1023_exact", "edge_1024_exact")] == [1023, 1024, 1023, 1024]
    starts = [r.start for r in EDGES["edge_out_of_phase"].rows]
    assert sum((s - min(starts)) % 160 != 0 for s in starts) == 1
    assert len({reduced(r, 48000) for r in EDGES["edge_second_rate_pair"].rates}) == 2
    for n, chunked in (("edge_clip_32767", False), ("edge_clip_32768", False), ("edge_clip_32769", True)):
        r = EDGES[n].rows[0]
        assert (min(r.span, 32768) < r.pcm.size) == chunked


def lerpmix_emu_lib():
    """librodio_b200_hostemu_lerpmix.so: the host-emulated library (tests/emu/build_emu.py) with tests/emu/lerpmix_hostemu.cpp in
    place of hostemu.cpp -- k_lerp_mix walked as the kernel walks it, every read checked."""
    emu = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
    sys.path[:0] = [emu]
    import build_emu
    build_emu.host_lib()                      # builds the objects shared with it: rb_api.cu, rb_lanes_batch.cu, the warp program
    objs = build_emu.variant_objects()
    uobjs = [os.path.join(build_emu.OBJ, f"host_{u}.o") for u in ("rb_api", "rb_lanes_batch")]
    src = os.path.join(emu, "lerpmix_hostemu.cpp")
    lib = os.path.join(emu, "librodio_b200_hostemu_lerpmix.so")
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in objs + uobjs + build_emu.HOST_DEPS + [src]):
        o = os.path.join(build_emu.OBJ, "host_lerpmix_hostemu.o")
        subprocess.check_call(build_emu.CXX + ["-I", os.path.join(emu, "mockcuda"), "-c", src, "-o", o])
        subprocess.check_call(build_emu.CXX + ["-shared"] + uobjs + [o] + objs + ["-o", lib])
    return lib


def test_designs_hold_on_the_emulator(built):
    """test_lerp_mix_rows, unchanged, against the host-emulated library whose k_lerp_mix walks every CTA as the kernel does and
    aborts on any read outside a row's input."""
    here = os.path.dirname(os.path.abspath(__file__))
    lib = lerpmix_emu_lib()
    code = ("import sys; sys.path[:0] = [%r, %r]; import rodio_b200._capi as c; c.LIB_PATH = %r; import pytest; "
            "sys.exit(pytest.main([%r, '-q', '-m', 'gpu', '-x', '-p', 'no:cacheprovider']))"
            % (os.path.dirname(here), here, lib, os.path.abspath(__file__) + "::test_lerp_mix_rows"))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=1800, cwd=os.path.dirname(here))
    assert r.returncode == 0 and f"{len(CASE_NAMES)} passed" in r.stdout, (r.stdout + r.stderr)[-3000:]
