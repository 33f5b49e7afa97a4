"""Generator sources in streaming sessions: SineWave / SignalGenerator chains (RB_FX_SIGNAL as effects[0]) whose samples the session
generates into their FIFOs itself (k_fifo_generate), with no pushes.  Every scenario runs a generator session and its pushed twin --
the same session whose generators are TestSources pushed with the oracle's generator samples -- with the same renders and controls,
and asks for the same bytes; where no control intervenes, both also equal the oracle's chains summed in the documented slot order
(tests/emu/layout_scenarios.py) and, within 1e-5 * peak, the oracle's sequential mixer.

    python tests/emu/generator_scenarios.py <scenario> ...
runs them on the host-emulated library; tests/test_session_generators.py runs them there and on the device."""
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]
if __name__ == "__main__":
    import build_emu                                  # noqa: E402
    import rodio_b200._capi as capi                   # noqa: E402
    capi.LIB_PATH = build_emu.HOST_LIB
import ctypes as C                                    # noqa: E402

import front_fx_scenarios as F                        # noqa: E402
import layout_scenarios as L                          # noqa: E402
import oracle                                         # noqa: E402
import rodio_b200 as rb                               # noqa: E402
from rodio_b200 import _capi as capi                  # noqa: E402
from helpers import assert_bit_exact                  # noqa: E402

MS = 1_000_000
HELD = capi.RB_SESSION_HELD
ENDLESS = rb.source.ENDLESS
SINE, TRI, SQUARE, SAW = capi.RB_SIGNAL_SINE, capi.RB_SIGNAL_TRIANGLE, capi.RB_SIGNAL_SQUARE, capi.RB_SIGNAL_SAWTOOTH


class GSrc(F.FSrc):
    """A generator source: SignalGenerator(rate, freq, fn), `.take(n)` (ENDLESS: the generator itself), then the push program `prog`
    and the chain variant `kind` of layout_scenarios.Src.  chain(pcm=None) is the generator session's chain; chain(pcm) the twin's,
    a TestSource of those samples."""

    def __init__(self, rate, freq, fn=SINE, n=ENDLESS, prog=(), **kw):
        kw.setdefault("frames", 0)
        super().__init__(1, rate, prog, **kw)
        self.freq, self.fn, self.n = float(np.float32(freq)), fn, n
        self.gen = True

    def chain(self, mix_ch, mix_rate, pcm=None, pre=None, pauses=()):
        if pcm is not None:
            return super().chain(mix_ch, mix_rate, pcm, pre)
        s = F.apply_prog(rb.SignalGenerator(self.rate, self.freq, self.fn).take(self.n), self.prog)
        pre = self.pre if pre is None else pre
        if self.kind == "front":
            s = rb.UniformSourceIterator(s.amplify(pre).low_pass(self.lp).amplify(self.mid), mix_ch, mix_rate)
            return s.amplify(self.gain) if self.gain is not None else s
        if self.kind == "pre":
            s = s.amplify(pre)
        s = rb.UniformSourceIterator(s, mix_ch, mix_rate)
        if self.lp:
            s = s.low_pass(self.lp)
        return s.amplify(self.gain) if self.gain is not None else s

    def samples(self, upto):
        """The generator's first min(n, upto) samples, from the oracle's literal generator."""
        return oracle.signal(self.fn, self.rate, self.freq, min(self.n, upto))


class PSrc(F.FSrc):
    """A pushed source beside the generators: the same in both sessions."""
    gen = False

    def samples(self, upto):
        return self.pcm


def sessions(srcs, mix_ch, mix_rate, block=480, fifo=2048, restarts=False, master=(), out_frames=None):
    """(generator session, twin, the twin's PCM per source).  The twin gets all of its PCM at once -- any split into pushes renders
    the same bytes: enough for out_frames mixer frames where a generator is endless (without out_frames: three seconds, which its
    take_duration ends first), and the end of stream where its `.take(n)` ends it.  Pushed sources get their PCM in both sessions."""
    starts = [s.start for s in srcs]
    pcms = []
    for s in srcs:
        want = 3 * s.rate if out_frames is None else int(math.ceil((out_frames + 64) * s.eff_rate() / mix_rate)) + 64
        pcms.append(s.samples(want) if s.gen else s.pcm)
    cap = max([fifo] + [p.size // s.ci + 64 for p, s in zip(pcms, srcs)])
    pushed = max([0] + [s.pcm.size // s.ci + 64 for s in srcs if not s.gen])
    gen = rb.Session([s.chain(mix_ch, mix_rate) for s in srcs], mix_rate, fifo_frames=max(fifo, pushed), max_block_frames=block,
                     mix_starts=starts, ctx=L.CTX["ctx"], mixer_channels=mix_ch, master=master, restarts=restarts)
    for i, s in enumerate(srcs):
        if not s.gen:
            gen.push(i, s.pcm, end_of_stream=True)
    twin = rb.Session([s.chain(mix_ch, mix_rate, p) for s, p in zip(srcs, pcms)], mix_rate, fifo_frames=cap, max_block_frames=block,
                      mix_starts=starts, ctx=L.CTX["ctx"], mixer_channels=mix_ch, master=master, restarts=restarts)
    for i, (s, p) in enumerate(zip(srcs, pcms)):
        twin.push(i, p, end_of_stream=not s.gen or s.n <= p.size)
    return gen, twin, pcms


def lockstep(gen, twin, rng, block, out_frames=None, hooks=None, what=""):
    """Render both with the same random block sizes (and the same controls: hooks[round](gen, twin) may return a new generator
    session) until both end or out_frames frames are out; each render must give the same frames on both."""
    got, ref, rnd, total = [], [], 0, 0
    while True:
        if hooks and rnd in hooks:
            r = hooks[rnd](gen, twin)
            gen = r if isinstance(r, rb.Session) else gen
        n = int(rng.integers(1, block + 1))
        if out_frames is not None:
            n = min(n, out_frames - total)
            if n == 0:
                break
        a, ea = gen.render(n)
        b, eb = twin.render(n)
        assert a.size == b.size and ea == eb, f"{what}: round {rnd}: {a.size} vs {b.size} samples, ended {ea} vs {eb}"
        got.append(a), ref.append(b)
        total += a.size // gen.channels
        rnd += 1
        if ea or (a.size == 0 and not (hooks and any(k > rnd for k in hooks))):
            break
        assert rnd < 200000
    got, ref = np.concatenate(got), np.concatenate(ref)
    assert_bit_exact(got, ref, what + ": against the pushed twin")
    return got, gen


def case(srcs, mix_ch, mix_rate, seed, what, block=480, out_frames=None, hooks=None, restarts=False, fifo=2048, oracle_check=True):
    gen, twin, pcms = sessions(srcs, mix_ch, mix_rate, block, fifo, restarts, out_frames=out_frames)
    got, gen = lockstep(gen, twin, np.random.default_rng(seed), block, out_frames, hooks, what)
    if oracle_check:
        real = [s.chain(mix_ch, mix_rate, p) for s, p in zip(srcs, pcms)]
        want = L.slot_expected(F.per_source(real, mix_ch, mix_rate), [s.start for s in srcs], srcs, mix_ch, mix_rate)
        assert_bit_exact(got, want[:got.size], what + ": against the oracle's chains in slot order")
        if out_frames is None:
            F.check(got, srcs, real, [s.start for s in srcs], mix_ch, mix_rate, what)
    runs = [(gen.source_runs(i), twin.source_runs(i)) for i in range(len(srcs))]
    gen.close(), twin.close()
    return got, runs


# ---------------------------------------------------------------------------------------------------------------------
def s_equivalence():
    """The four functions at 48, 44.1, 22.05 and 96 kHz into mixers of 1, 2 and 6 channels, endless and `.take(n)`, a frequency above
    the rate (step >= 1), the three chain variants, random block splits."""
    rates = (48000, 44100, 22050, 96000)
    for m, mix_ch in enumerate((1, 2, 6)):
        srcs = []
        for k in range(8):
            rate = rates[(k + m) % 4]
            freq = (440.0, 1234.5, 97.25, 70000.0, 3000.0, 55.0, 23456.0, 7.5)[k]
            kind = ("behind", "pre", "front", "behind")[k % 4] if mix_ch > 1 or k % 4 != 2 else "behind"
            n = ENDLESS if k % 3 else 1500 + 101 * k
            srcs.append(GSrc(rate, freq, fn=k % 4, n=n, kind=kind, lp=None if k % 2 else 900, start=(53 * k) % 150, seed=k))
        case(srcs, mix_ch, 48000, 3 + m, f"{mix_ch}-channel mixer", block=333, out_frames=2500)
    # .take(n) only: the sessions end, and equal the oracle's mixer
    srcs = [GSrc(r, f, fn=k % 4, n=700 + 61 * k, start=17 * k, seed=k) for k, (r, f) in enumerate([(44100, 440.0), (22050, 30000.0), (96000, 880.0), (48000, 48000.0)])]
    case(srcs, 2, 48000, 9, "finite generators")


def s_examples():
    """The rodio example shapes: basic.rs (held generators started at chosen frames), mix_multiple_sources.rs (four sines from frame 0),
    distortion.rs (amplify, distortion and take_duration in the program), take_duration with filter_fadeout and fade_in, and resampled
    1 s takes with RB_SESSION_RESTARTS (several converter runs, counted as for the pushed twin)."""
    d = lambda ms: ms * MS
    four = [GSrc(48000, f, prog=[("amp", 0.1), ("take", d(60), False)], kind="behind", lp=None, gain=None, seed=k)
            for k, f in enumerate((440.0, 220.0, 660.0, 880.0))]
    case(four, 2, 48000, 1, "mix_multiple_sources.rs")
    basic = [GSrc(48000, 740.0, prog=[("amp", 0.1), ("take", d(40), False)], kind="behind", lp=None, gain=None, start=HELD, seed=1),
             GSrc(48000, 440.0, prog=[("amp", 0.2), ("take", d(30), False)], kind="behind", lp=None, gain=None, start=HELD, seed=2),
             GSrc(48000, 220.0, prog=[("amp", 0.05)], kind="behind", lp=None, gain=None, seed=3, n=5000)]

    def start(i):
        return lambda g, t: (g.start(i), t.start(i))
    case(basic, 2, 48000, 2, "basic.rs", block=240, hooks={3: start(0), 7: start(1)}, oracle_check=False)
    dist = [GSrc(48000, 440.0, prog=[("amp", 0.9), ("dist", 4.0, 0.5), ("take", d(50), False)], lp=None, gain=None, seed=1),
            GSrc(44100, 220.0, fn=TRI, prog=[("dist", 2.5, 0.3), ("take", d(45), True)], lp=800, seed=2),
            GSrc(48000, 330.0, prog=[("fade_in", d(20)), ("take", d(55), True)], kind="pre", pre=0.7, lp=None, seed=3)]
    case(dist, 2, 48000, 4, "distortion.rs, fade_in, filter_fadeout")
    # SineWave at 48 kHz, take_duration(1 s) into a 44.1 kHz mixer: two converter runs (32768 + 15232 samples)
    takes = [GSrc(48000, 440.0 + 37 * k, prog=[("amp", 0.2), ("take", 1000 * MS, False)], lp=None if k % 2 else 2000, seed=k) for k in range(3)]
    _, runs = case(takes, 2, 44100, 5, "resampled 1 s takes", block=480, restarts=True)
    assert all(a == b == 2 for a, b in runs), runs


def s_controls():
    """skip ends an endless generator after the converter's last pulled frame and a source queued behind it starts next; `ended`
    only once nothing endless is left; set_volume / set_amplify mid-play; generators and pushed sources in one class."""
    a = GSrc(44100, 440.0, kind="pre", pre=0.5, lp=700, seed=1)                        # endless, skipped at round 6
    b = GSrc(44100, 660.0, fn=SAW, n=3000, kind="pre", pre=0.8, lp=700, start=HELD, seed=2)   # queued behind a
    c = PSrc(1, 44100, kind="pre", pre=0.9, lp=700, frames=6000, seed=3)              # pushed, in a's class
    e = GSrc(22050, 300.0, fn=SQUARE, kind="behind", lp=None, seed=4)                  # endless, skipped at round 14

    def skip(i):
        return lambda g, t: (g.skip(i), t.skip(i))

    def controls(g, t):
        for x in (g, t):
            x.set_volume(0, 0.25), x.set_amplify(2, 1.5), x.set_amplify(3, 0.5)
        n, ended = g.available()
        assert n > 0 and not ended

    def queue(g, t):
        g.follow(1, 0), t.follow(1, 0)

    def check_alive(g, t):
        assert not g.available()[1]
    hooks = {0: queue, 4: controls, 6: skip(0), 10: check_alive, 14: skip(3)}
    got, _ = case([a, b, c, e], 2, 48000, 6, "skip, follow, volume, a shared class", block=400, hooks=hooks, oracle_check=False)
    # an endless generator alone never ends by itself
    gen, twin, _ = sessions([GSrc(48000, 1000.0, seed=0)], 1, 48000, out_frames=5000)
    got, gen = lockstep(gen, twin, np.random.default_rng(1), 480, out_frames=5000, what="endless")
    assert got.size == 5000 and not gen.available()[1]
    gen.skip(0)
    while True:
        x, ended = gen.render(480)
        if ended or x.size == 0:
            break
    assert ended
    gen.close(), twin.close()


def s_state():
    """A mid-play get_state -> set_state hand-over to a fresh session continues bit for bit; blobs are refused across generator
    sets; sessions without generators keep their blob versions."""
    srcs = [GSrc(44100, 440.0, kind="pre", pre=0.7, seed=1), GSrc(48000, 523.25, fn=TRI, prog=[("fade_in", 30 * MS)], seed=2),
            PSrc(2, 22050, frames=4000, seed=3), GSrc(96000, 1500.0, fn=SAW, n=9000, seed=4)]
    mk = lambda: sessions(srcs, 2, 48000, out_frames=0)[0]
    blobs = {}

    def hand_over(g, t):
        blob = g.get_state()
        assert int.from_bytes(blob[4:8], "little") == 10
        blobs["mid"] = blob
        n = mk()
        n.set_state(blob)
        g.close()
        return n
    case(srcs, 2, 48000, 7, "hand-over", hooks={5: hand_over}, out_frames=4000, oracle_check=False)
    blob = blobs["mid"]
    others = [[GSrc(44100, 441.0, kind="pre", pre=0.7, seed=1)] + srcs[1:],                         # another frequency
              [GSrc(44100, 440.0, fn=SQUARE, kind="pre", pre=0.7, seed=1)] + srcs[1:],              # another function
              srcs[:3] + [GSrc(96000, 1500.0, fn=SAW, n=9001, seed=4)],                              # another take(n)
              [PSrc(1, 44100, kind="pre", pre=0.7, seed=1)] + srcs[1:]]                             # a pushed source in its place
    for o in others:
        with sessions(o, 2, 48000, out_frames=0)[0] as s:
            st = capi.lib().rb_session_set_state(s._h, (C.c_uint8 * len(blob)).from_buffer_copy(blob), len(blob))
            assert st == capi.RB_ERR_INVALID_ARGUMENT, st
    plain = [PSrc(1, 44100, kind="pre", pre=0.7, seed=1), PSrc(2, 22050, frames=4000, seed=3)]
    with sessions(plain, 2, 48000, out_frames=0)[0] as s:
        b = s.get_state()
        assert int.from_bytes(b[4:8], "little") in (5, 6)
        st = capi.lib().rb_session_set_state(s._h, (C.c_uint8 * len(blob)).from_buffer_copy(blob), len(blob))
        assert st == capi.RB_ERR_INVALID_ARGUMENT, st
        with sessions(srcs, 2, 48000, out_frames=0)[0] as g:
            st = capi.lib().rb_session_set_state(g._h, (C.c_uint8 * len(b)).from_buffer_copy(b), len(b))
            assert st == capi.RB_ERR_INVALID_ARGUMENT, st


def soak(seconds):
    """`seconds` of 10 ms blocks: the f32 phase carries from fill to fill exactly as it drifts in the generator."""
    srcs = [GSrc(48000, 440.0, lp=None, gain=None, seed=1), GSrc(44100, 997.0, fn=TRI, seed=2), GSrc(48000, 47000.0, fn=SAW, seed=3)]
    frames = 48000 * seconds
    gen, twin, _ = sessions(srcs, 1, 48000, block=480, out_frames=frames)
    got, ref = [], []
    for _ in range(frames // 480):
        a, _ = gen.render(480)
        b, _ = twin.render(480)
        got.append(a), ref.append(b)
    assert_bit_exact(np.concatenate(got), np.concatenate(ref), f"{seconds} s soak")
    gen.close(), twin.close()


def s_soak():
    soak(30)


def s_errors():
    """A generator takes no pushes: push / push_spans with frames, end_of_stream or marks and push_packed(_spans) with a count, an
    end of stream or a mark for it are RB_ERR_STATE, push_silence is RB_ERR_UNSUPPORTED; none of them changes what renders.  Creation
    validates a generator as rb_stream_plan does."""
    lib = capi.lib()
    srcs = [GSrc(44100, 440.0, seed=1), PSrc(1, 44100, frames=3000, seed=2)]
    gen, twin, _ = sessions(srcs, 2, 48000, restarts=True, out_frames=3000)
    x = np.zeros(64, np.float32)
    p = x.ctypes.data_as(C.c_void_p)
    mark = (capi.rb_span_mark * 1)(capi.rb_span_mark(0, 0, 0))
    assert lib.rb_session_push(gen._h, 0, p, 64, 0) == capi.RB_ERR_STATE
    assert lib.rb_session_push(gen._h, 0, p, 0, 1) == capi.RB_ERR_STATE
    assert lib.rb_session_push_spans(gen._h, 0, p, 64, None, 0, 0) == capi.RB_ERR_STATE
    assert lib.rb_session_push_spans(gen._h, 0, p, 0, mark, 1, 0) == capi.RB_ERR_STATE
    for counts, eos, marks in (((64, 0), None, None), ((0, 0), (1, 0), None), ((0, 0), None, (1, 0))):
        n = (C.c_uint64 * 2)(*counts)
        e = (C.c_uint8 * 2)(*eos) if eos else None
        if marks is None:
            assert lib.rb_session_push_packed(gen._h, p, n, e) == capi.RB_ERR_STATE
        else:
            assert lib.rb_session_push_packed_spans(gen._h, p, n, e, (C.c_uint32 * 2)(*marks), mark) == capi.RB_ERR_STATE
    assert lib.rb_session_push_silence(gen._h, 0, 64) == capi.RB_ERR_UNSUPPORTED
    assert lib.rb_session_push(gen._h, 0, p, 0, 0) == capi.RB_OK
    gen.push_packed([x, np.zeros(0, np.float32)], [True, False])   # the helper passes the generator by
    got, gen = lockstep(gen, twin, np.random.default_rng(2), 480, out_frames=3000, what="after refusals")
    gen.close(), twin.close()
    # creation: the batch rules for a generator descriptor, statuses as rb_stream_plan gives them
    base = rb.UniformSourceIterator(rb.SineWave(440.0).amplify(0.5), 1, 48000)
    variants = []
    for field, value in (("n_samples", 4), ("channels", 2), ("span_len", 7), ("format", capi.RB_FMT_I16)):
        variants.append(("desc", field, value))
    for u32, f32 in ((7, 440.0), (0, 0.0), (0, -3.0), (0, float("inf")), (0, float("nan"))):
        variants.append(("fx", u32, f32))
    for v in variants:
        descs, keep = rb.source.pack_descs([base], [0])
        if v[0] == "desc":
            setattr(descs[0], v[1], v[2])
        else:
            keep[1][0].u32[0], keep[1][0].f32[0] = v[1], v[2]
        h = C.c_void_p()
        want = lib.rb_stream_plan(C.byref(descs[0]), 1, 48000, None, None, None, None)
        got = lib.rb_session_create(L.CTX["ctx"]._h if L.CTX["ctx"] else rb.default_context()._h, 1, 48000, descs, 1, 1024, 480, C.byref(h))
        assert want != capi.RB_OK and got == want, (v, got, want)


SCENARIOS = {"equivalence": s_equivalence, "examples": s_examples, "controls": s_controls, "state": s_state, "soak": s_soak,
             "errors": s_errors}

if __name__ == "__main__":
    for name in (sys.argv[1:] or list(SCENARIOS)):
        SCENARIOS[name]()
        print("ok", name, flush=True)
