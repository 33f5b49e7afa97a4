"""Restart schedules of the streaming sessions (rb_session_create_ex with RB_SESSION_RESTARTS): the mixer's conversion ends one
SampleRateConverter run and begins the next where rodio's UniformSourceIterator does -- every min(span_len, 32768) samples of a
source that reports a span, and every min(samples left, 32768) behind take_duration, a pause's zeros counted.  Every scenario
compares the session's output bit for bit with the oracle's literal chains (which restart by themselves) summed in the documented
slot order, and within 1e-5 * peak with the oracle's sequential mixer; it asserts through rb_session_source_runs that the runs it
designed were started and through rb_session_restart_launches that only blocks with a restart took the RESTART kernels.

    python tests/emu/restart_scenarios.py <scenario> ...
runs them on the host-emulated library; tests/test_session_restarts.py runs them there and on the device."""
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
import front_fx_scenarios as F                        # noqa: E402
import rodio_b200 as rb                               # noqa: E402
from rodio_b200 import _capi as capi                  # noqa: E402

L = F.L
MS = F.MS
HELD = capi.RB_SESSION_HELD
CAP = 32768


class RSrc(F.FSrc):
    """A front-fx source whose base reports current_span_len() = Some(span) at every bootstrap (0: None; 'len': a SamplesBuffer,
    which reports its length)."""

    def __init__(self, ci, rate, prog=(), span=0, **kw):
        super().__init__(ci, rate, prog, **kw)
        self.span = self.pcm.size if span == "len" else span

    def chain(self, mix_ch, mix_rate, pcm=None, pre=None, pauses=(), gain=None):
        pcm = np.zeros(0, np.float32) if pcm is None else pcm
        s = F.apply_prog(rb.Source(pcm, self.ci, self.rate, span_len=self.span), self.prog)
        if pauses:
            s = s.speed(1.0)
            shift = 0
            for at, frames in pauses:
                s = s.pause_at(at + shift, frames)
                shift += frames * self.ci
        pre = self.pre if pre is None else pre
        gain = self.gain if gain is None else gain
        if self.kind == "front":
            s = rb.UniformSourceIterator(s.amplify(pre).low_pass(self.lp).amplify(self.mid), mix_ch, mix_rate)
            return s.amplify(gain) if gain is not None else s
        if self.kind == "pre":
            s = s.amplify(pre)
        s = rb.UniformSourceIterator(s, mix_ch, mix_rate)
        if self.lp:
            s = s.low_pass(self.lp)
        return s.amplify(gain) if gain is not None else s

    def frames(self):
        return self.pcm.size // self.ci

    def run_frames(self):
        """Frames per run from the span alone (no take); None: one run."""
        return min(self.span, CAP) // self.ci if self.span else None


def session(srcs, mix_ch, mix_rate, starts=None, fifo=4096, block=480, restarts=True):
    return rb.Session([s.chain(mix_ch, mix_rate) for s in srcs], mix_rate, fifo_frames=fifo, max_block_frames=block,
                      mix_starts=starts if starts is not None else [s.start for s in srcs], ctx=L.CTX["ctx"], mixer_channels=mix_ch,
                      restarts=restarts)


def out_total(n, f, t):
    if n < 2:
        return n
    ns = ((n - 1) * t + f - 1) // f
    return ns + (1 if ns * f < n * t else 0)


def pulled_after(runs, f, t, n_out):
    """Input frames the converter has pulled once n_out outputs were rendered, for run lengths `runs` (frames)."""
    i = o = 0
    for n in runs:
        tot = out_total(n, f, t)
        if n_out <= o + tot:
            return i + min(((n_out - 1 - o) * f) // t + 2, n) if n_out > o else i
        i, o = i + n, o + tot
    return i


def ratio(rate, mix_rate):
    g = math.gcd(rate, mix_rate)
    return rate // g, mix_rate // g


def span_runs(s, mix_rate, n=None):
    """Run lengths of source s over its first n frames (the span schedule)."""
    n = s.frames() if n is None else n
    r = s.run_frames()
    if r is None or s.rate == mix_rate:
        return [n]
    return [min(r, n - a) for a in range(0, n, r)]


def drive(sess, srcs, rng=None, push=None, block=480, pauses=None, hooks=None, packed=True):
    """Push push[i] frames per source and round (random 0 .. 2 push[i] with rng), silence at pauses[i] = [(frame, frames), ...],
    render until nothing comes.  hooks[rnd](sess, mixer frames so far) may return a new session."""
    push = push or [max(1, s.rate // 100) for s in srcs]
    pos, got, ended, rnd = [0] * len(srcs), [], False, 0
    todo = [list(p) for p in (pauses or [[]] * len(srcs))]
    mix_ch = sess.channels
    while not ended:
        if hooks and rnd in hooks:
            r = hooks[rnd](sess, sum(b.size for b in got) // mix_ch)
            sess = r if r is not None else sess
        blocks, eos, silence = [], [], []
        for i, s in enumerate(srcs):
            k = min(int(rng.integers(0, 2 * push[i] + 1)) if rng is not None else push[i], s.frames() - pos[i])
            if todo[i] and pos[i] <= todo[i][0][0] <= pos[i] + k:
                k = todo[i][0][0] - pos[i]
                silence.append((i, todo[i].pop(0)[1]))
            blocks.append(s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)])
            pos[i] += k
            eos.append(pos[i] == s.frames() and not todo[i])
        if packed:
            sess.push_packed(blocks, eos)
        else:
            for i, (b, e) in enumerate(zip(blocks, eos)):
                if b.size or e:
                    sess.push(i, b, end_of_stream=e)
        for i, n in silence:
            sess.push_silence(i, n)
        while True:
            b, ended = sess.render(int(rng.integers(1, block + 1)) if rng is not None else block)
            got.append(b)
            if b.size == 0 or ended:
                break
        rnd += 1
        assert rnd < 200000
    return np.concatenate(got), sess


def hand_over(srcs, mix_ch, mix_rate, **kw):
    def swap(sess, _):
        t = session(srcs, mix_ch, mix_rate, **kw)
        t.set_state(sess.get_state())
        sess.close()
        return t
    return swap


def run(srcs, mix_ch, mix_rate, seed, what, block=480, swap_at=None, pauses=None, fifo=4096, packed=True, split=True):
    sess = session(srcs, mix_ch, mix_rate, block=block, fifo=fifo)
    hooks = {swap_at: hand_over(srcs, mix_ch, mix_rate, block=block, fifo=fifo)} if swap_at is not None else None
    got, sess = drive(sess, srcs, np.random.default_rng(seed) if split else None, block=block, pauses=pauses, hooks=hooks, packed=packed)
    runs = [sess.source_runs(i) for i in range(len(srcs))]
    launches = sess.restart_launches()
    sess.close()
    real = [s.chain(mix_ch, mix_rate, s.pcm, pauses=[(at * s.ci, n) for at, n in (pauses[i] if pauses else [])]) for i, s in enumerate(srcs)]
    F.check(got, srcs, real, [s.start for s in srcs], mix_ch, mix_rate, what)
    return runs, launches


# ---------------------------------------------------------------------------------------------------------------------
VARIANTS = [dict(lp=None, gain=None), dict(lp=None, gain=0.8), dict(lp=700, gain=None), dict(kind="pre", pre=0.6), dict(kind="front", gain=None),
            dict(kind="front", gain=0.9)]


def s_spans():
    """span_len = the source's length (a SamplesBuffer), 2304 (a packet), 32768, 65536 and 4 (sub-blocks); mono, stereo, 4- and
    8-channel sources in 2-, 6- and 8-channel mixers; up-, same-rate and down-sampling; every chain variant; a hand-over."""
    for m, mix_ch in enumerate((2, 6, 8)):
        srcs = []
        for k, (ci, rate, span, frames) in enumerate([(2, 44100, 2304, 5000), (1, 44100, 2304, 5000), (2, 96000, 2304, 7000), (2, 48000, 2304, 3000),
                                                      (4, 44100, 2304, 2500), (8, 22050, 2304, 1500), (2, 44100, "len", 3000), (2, 96000, 4, 300),
                                                      (1, 44100, 4, 300), (2, 44100, 65536, 17500), (2, 44100, 32768, 17000), (1, 96000, 32768, 34000),
                                                      (2, 44100, 0, 2000)]):
            if m and frames > 10000:
                continue
            srcs.append(RSrc(ci, rate, span=span, frames=frames, start=0 if k % 3 else 7 * k, seed=2000 + 100 * m + k, **VARIANTS[(k + m) % len(VARIANTS)]))
        runs, launches = run(srcs, mix_ch, 48000, 31 + m, f"spans, {mix_ch}-channel mixer", swap_at=3, block=333 if m else 480, fifo=16384)
        for i, s in enumerate(srcs):
            assert runs[i] == len(span_runs(s, 48000)), (i, runs[i], len(span_runs(s, 48000)))
        assert launches > 0
    # the same sources without the flag, or with it and no span: no RESTART launch, one run each
    srcs = [RSrc(2, 44100, span=s, frames=3000, seed=2900 + k, **VARIANTS[k]) for k, s in enumerate((2304, 0, "len"))]
    for restarts, spans in ((False, None), (True, 0)):
        use = srcs if spans is None else [RSrc(2, 44100, span=0, frames=3000, seed=2900 + k, **VARIANTS[k]) for k in range(3)]
        sess = session(use, 2, 48000, restarts=restarts)
        got, sess = drive(sess, use, np.random.default_rng(3))
        assert sess.restart_launches() == 0 and [sess.source_runs(i) for i in range(3)] == [1, 1, 1]
        sess.close()
        one_run = [RSrc(2, 44100, span=0, frames=3000, seed=2900 + k, **VARIANTS[k]) for k in range(3)]
        F.check(got, one_run, [s.chain(2, 48000, s.pcm) for s in one_run], [0, 0, 0], 2, 48000, "no schedule")


def take_of(rate, ci, samples, fade=True):
    return ("take", samples * (10**9 // (rate * ci)), fade)


def s_takes():
    """44.1 kHz stereo clips behind fade_in.take_duration(.., fade-out filter) of 350 ms, one frame over a run, 1.5 s and 3 s; a pause
    before, across and after a run boundary."""
    ms = lambda t: 2 * (44100 * t // 1000)
    takes = [ms(350), CAP + 2, ms(1500), ms(3000), ms(1500), ms(1500), ms(1500)]
    srcs = [RSrc(2, 44100, [("fade_in", 200 * MS), take_of(44100, 2, n)], kind="pre", pre=1.0, lp=None if k % 2 else 700, frames=n // 2 + 500,
                 seed=3000 + k) for k, n in enumerate(takes)]
    pauses = [[], [], [], [], [(16000, 300)], [(16300, 400)], [(16384 + 200, 250), (40000, 64)]]
    runs, launches = run(srcs, 2, 48000, 41, "takes", swap_at=40, pauses=pauses, split=False, fifo=8192)
    want = [1, 2, 5, 9]
    assert runs[:4] == want and all(r >= 5 for r in runs[4:]) and launches > 0, (runs, launches)


def s_split_invariance():
    """1- to 7-frame pushes and renders against the bytes of a one-block render; pushes that end one frame before, on and after a
    run's last input frame with a render after each (starved exactly at the cut); end of stream inside the first two frames of a run."""
    specs = [(2, 44100, 40, 700, VARIANTS[2]), (1, 44100, 24, 650, VARIANTS[3]), (2, 96000, 2304, 2400, VARIANTS[4]), (2, 22050, 64, 321, VARIANTS[1]),
             (4, 44100, 80, 401, VARIANTS[0]), (2, 48000, 40, 500, VARIANTS[2])]
    srcs = [RSrc(ci, r, span=sp, frames=fr, seed=4000 + k, **v) for k, (ci, r, sp, fr, v) in enumerate(specs)]
    sess = session(srcs, 6, 48000, block=8192)
    for i, s in enumerate(srcs):
        sess.push(i, s.pcm, end_of_stream=True)
    whole, done = [], False
    while not done:
        b, done = sess.render(8192)
        whole.append(b)
    whole = np.concatenate(whole)
    assert [sess.source_runs(i) for i in range(len(srcs))] == [len(span_runs(s, 48000)) for s in srcs]
    sess.close()
    F.check(whole, srcs, [s.chain(6, 48000, s.pcm) for s in srcs], [0] * len(srcs), 6, 48000, "one-block render")
    for packed in (True, False):
        sess = session(srcs, 6, 48000, block=512)
        got, sess = drive(sess, srcs, np.random.default_rng(5), push=[3] * len(srcs), block=11, packed=packed)
        sess.close()
        assert np.array_equal(got.view(np.uint32), whole.view(np.uint32)), f"split (packed={packed}) differs from the one-block render"
    # around one cut, frame by frame: runs of 20 frames; the input ends 0, 1 and 2 frames into the third run
    for tail in (0, 1, 2):
        s = RSrc(2, 44100, span=40, frames=40 + tail, seed=4100 + tail, **VARIANTS[2])
        sess = session([s], 2, 48000, block=64)
        got, pos = [], 0
        for k in (18, 1, 1, 1, 1, 17, 1, 1, 1, 1):
            k = min(k, s.frames() - pos)
            sess.push(0, s.pcm[2 * pos: 2 * (pos + k)], end_of_stream=(pos + k == s.frames()))
            pos += k
            while True:
                b, ended = sess.render(64)
                got.append(b)
                if b.size == 0 or ended:
                    break
        assert ended and sess.source_runs(0) == 2 + (tail > 0)
        sess.close()
        F.check(np.concatenate(got), [s], [s.chain(2, 48000, s.pcm)], [0], 2, 48000, f"frame by frame around a cut, tail {tail}")


def s_controls():
    """set_volume and set_amplify in the blocks around a cut (a gain in front and the volume behind a filter in front), a source
    queued behind one with a schedule, skip inside a run, a state hand-over with a cut in the next block, and a blob offered to a
    session with another schedule."""
    mix_ch, mix_rate, block = 2, 48000, 100
    srcs = [RSrc(2, 44100, span=800, frames=3000, kind="pre", pre=1.0, lp=700, seed=5000),
            RSrc(2, 44100, span=800, frames=3000, lp=700, gain=1.0, seed=5001),
            RSrc(1, 22050, span=300, frames=900, kind="pre", pre=1.0, seed=5002),
            RSrc(2, 44100, span=800, frames=3000, kind="pre", pre=1.0, seed=5003)]
    starts = [0, 0, HELD, 0]
    fresh = lambda: session(srcs, mix_ch, mix_rate, starts=starts, block=block)
    sess = fresh()
    sess.follow(2, 0)
    for i, s in enumerate(srcs):
        sess.push(i, s.pcm[:2 * 2000] if i == 3 else s.pcm, end_of_stream=(i != 3))   # source 3 is skipped inside its third run
    f, t = ratio(44100, mix_rate)
    cut = out_total(400, f, t)                        # the first output of the second run (runs of 400 frames)
    got, marks, n, ended = [], {}, 0, False
    # blocks that end 30 frames before the cut, on it and 30 behind it, with a change after each; a hand-over 10 frames in front of
    # the next cut; a skip
    for upto, act in ((cut - 30, "vol"), (cut, "amp"), (cut + 30, "vol2"), (2 * cut - 10, "swap"), (2 * cut + 300, "skip"), (None, None)):
        while not ended and (upto is None or n < upto):
            b, ended = sess.render(block if upto is None else min(block, upto - n))
            got.append(b)
            n += b.size // mix_ch
            if b.size == 0:
                break
        marks[act] = n
        if act == "vol":
            sess.set_volume(0, 0.5)
        elif act == "amp":
            sess.set_amplify(1, 0.25)
        elif act == "vol2":
            sess.set_volume(0, 1.5)
        elif act == "swap":
            blob = sess.get_state()
            assert int.from_bytes(blob[4:8], "little") == 8
            t2 = fresh()
            t2.set_state(blob)
            sess.close()
            sess = t2
        elif act == "skip":
            sess.skip(3)
    assert ended
    runs = [sess.source_runs(i) for i in range(4)]
    sess.close()
    got = np.concatenate(got)
    # expected: a frame keeps the factor of the block that pulled it; the gain behind changes with the block; the skipped source
    # ends with the last frame the converter pulled
    r400 = span_runs(srcs[0], mix_rate)
    p1, p2 = pulled_after(r400, f, t, marks["vol"]), pulled_after(r400, f, t, marks["vol2"])
    vol = np.ones(3000, np.float32)
    vol[p1:p2], vol[p2:] = 0.5, 1.5
    p_skip = pulled_after(span_runs(srcs[3], mix_rate, 2000), f, t, marks["skip"])
    real = [s.chain(mix_ch, mix_rate, s.pcm) for s in srcs]
    real[0] = srcs[0].chain(mix_ch, mix_rate, (srcs[0].pcm.reshape(-1, 2) * vol[:, None]).reshape(-1))
    real[3] = srcs[3].chain(mix_ch, mix_rate, srcs[3].pcm[:2 * p_skip])
    per = F.per_source(real, mix_ch, mix_rate)
    quarter = F.per_source([srcs[1].chain(mix_ch, mix_rate, srcs[1].pcm, gain=0.25)], mix_ch, mix_rate)[0]
    per[1] = np.concatenate([per[1][:mix_ch * marks["amp"]], quarter[mix_ch * marks["amp"]:]])
    want = L.slot_expected(per, [0, 0, per[0].size // mix_ch, 0], srcs, mix_ch, mix_rate)
    F.assert_bit_exact(got, want[:got.size], "controls around a cut")
    assert got.size == want.size or not np.any(want[got.size:]), "tail"
    assert runs == [len(r400), len(r400), 3, len(span_runs(srcs[3], mix_rate, p_skip))], runs
    # the volume behind a filter in front of the conversion, changed on a cut: a tap keeps the factor it was pulled with
    s4 = RSrc(2, 44100, span=800, frames=1500, kind="front", pre=1.0, mid=1.0, gain=None, seed=5004)
    sess = session([s4], mix_ch, mix_rate, block=block)
    sess.push(0, s4.pcm, end_of_stream=True)
    got, n, ended = [], 0, False
    while not ended:
        b, ended = sess.render(min(block, cut - n) if n < cut else block)
        got.append(b)
        n += b.size // mix_ch
        if n == cut:
            sess.set_volume(0, 0.5)
    sess.close()
    got = np.concatenate(got)
    a, b = (F.per_source([RSrc(2, 44100, span=800, frames=1500, kind="front", pre=1.0, mid=v, gain=None, seed=5004).chain(mix_ch, mix_rate, s4.pcm)],
                         mix_ch, mix_rate)[0] for v in (1.0, 0.5))
    F.assert_bit_exact(got, np.concatenate([a[:mix_ch * cut], b[mix_ch * cut:]]) + np.float32(0.0), "volume behind a filter in front, changed on a cut")
    # a blob only loads into a session with the same schedules
    other = [RSrc(s.ci, s.rate, span=s.span + 2 * s.ci, frames=10, kind=s.kind, lp=s.lp, gain=s.gain, pre=s.pre) for s in srcs]
    for make in (lambda: session(other, mix_ch, mix_rate, starts=starts, block=block),
                 lambda: session(srcs, mix_ch, mix_rate, starts=starts, block=block, restarts=False)):
        with make() as t3:
            try:
                t3.set_state(blob)
            except capi.RodioB200Error as e:
                assert e.status == capi.RB_ERR_INVALID_ARGUMENT
            else:
                raise AssertionError("a blob with another schedule was accepted")


def s_refusals():
    """Runs that are not whole frames of the source, runs shorter than two frames, unknown flags; without the flag the refusals of
    before stand; blob versions of sessions without a schedule are those of before."""
    U, I = capi.RB_ERR_UNSUPPORTED, capi.RB_ERR_INVALID_ARGUMENT
    z = np.zeros(0, np.float32)

    def refused(make, status=U):
        try:
            make().close()
        except capi.RodioB200Error as e:
            assert e.status == status, e
        else:
            raise AssertionError("accepted")
    mk = lambda s, ch=2, restarts=True: rb.Session([rb.UniformSourceIterator(s, ch, 48000)], 48000, mixer_channels=ch, restarts=restarts)
    S = lambda ci, rate, span: rb.Source(z, ci, rate, span_len=span)
    refused(lambda: mk(S(2, 44100, 2305)))                       # not a multiple of the channel count
    refused(lambda: mk(S(3, 44100, 3 * 20000), 6))               # capped at 32768: not whole frames of three channels
    refused(lambda: mk(S(6, 48000, 6 * 20000), 6))               # ... at the mixer's rate as well: the channel conversion restarts inside a frame
    refused(lambda: mk(S(2, 44100, 2)))                          # one-frame runs
    refused(lambda: mk(S(3, 44100, 0).take_duration(F.take_ns(44100, 3, 1000)), 6))     # a long take of three channels
    refused(lambda: mk(S(2, 44100, 0).take_duration(F.take_ns(44100, 2, 20, whole=False))))   # a resampled take that ends inside a frame
    refused(lambda: mk(S(2, 44100, 0).take_duration(F.take_ns(44100, 2, 1000)), restarts=False))   # without the flag: as before
    mk(S(3, 44100, 3 * 700), 6).close()
    mk(S(2, 44100, 0).take_duration(F.take_ns(44100, 2, 1000))).close()
    mk(S(2, 44100, 2305), restarts=False).close()                # without the flag span_len is ignored
    import ctypes as C
    d, keep = rb.source.pack_descs([rb.UniformSourceIterator(S(2, 44100, 0), 2, 48000)], None)
    h = C.c_void_p()
    ctx = L.CTX["ctx"] or rb.source.default_context()
    assert capi.lib().rb_session_create_ex(ctx._h, 2, 48000, d, 1, 4096, 480, 2, C.byref(h)) == I
    with mk(S(2, 44100, 0)) as s:                                 # the flag alone adds no schedule: version 5
        assert int.from_bytes(s.get_state()[4:8], "little") == 5
    with mk(S(2, 44100, 2304)) as s:
        assert int.from_bytes(s.get_state()[4:8], "little") == 8 and s.source_runs(0) == 0 and s.restart_launches() == 0
        try:
            s.source_runs(1)
        except capi.RodioB200Error as e:
            assert e.status == I
        else:
            raise AssertionError("source index out of range accepted")


def soak(seed, cases):
    """Random schedules: spans, rates, layouts, chain variants, takes with pauses, random splits."""
    rng = np.random.default_rng(seed)
    for case in range(cases):
        mix_ch = int(rng.choice([1, 2, 2, 6]))
        mix_rate = int(rng.choice([48000, 44100]))
        srcs, pauses = [], []
        for k in range(int(rng.integers(1, 9))):
            ci = 1 if mix_ch == 1 else int(rng.choice([1, 2, 2, 4]))
            rate = int(rng.choice([44100, 22050, 48000, 96000, 32000]))
            frames = int(rng.integers(1, 1500))
            span = ci * int(rng.choice([0, 2, 3, 5, 17, 100, 1152, int(rng.integers(2, 900))]))
            v = dict(VARIANTS[int(rng.integers(len(VARIANTS)))])
            prog, p = [], []
            if rng.random() < 0.3 and v.get("kind") != "front":
                take = ci * int(rng.integers(2, frames + 2))
                fade = bool(rng.random() < 0.5) and take * 1000 >= 2 * rate * ci      # rodio's fade-out divides by the take's whole milliseconds
                prog = [("fade_in", 3 * MS), take_of(rate, ci, take, fade)]
                if rng.random() < 0.5:
                    p = [(int(rng.integers(0, min(frames, take // ci))), int(rng.integers(1, 200)))]
            srcs.append(RSrc(ci, rate, prog, span=span, frames=frames, start=0 if rng.random() < 0.6 else int(rng.integers(0, 300)),
                             seed=90000 + 100 * case + k + 7919 * seed, **v))
            pauses.append(p)
        try:
            run(srcs, mix_ch, mix_rate, 1000 * seed + case, f"soak seed {seed} case {case}", block=int(rng.choice([7, 64, 480])), pauses=pauses,
                swap_at=int(rng.integers(0, 6)) if rng.random() < 0.5 else None, packed=bool(rng.random() < 0.5), fifo=2048)
        except Exception:
            print("soak seed", seed, "case", case, [(s.ci, s.rate, s.span, s.frames(), s.kind, s.lp, s.gain, s.prog, s.start) for s in srcs], pauses, flush=True)
            raise


def s_soak():
    soak(1, 12)


SCENARIOS = {"spans": s_spans, "takes": s_takes, "split_invariance": s_split_invariance, "controls": s_controls, "refusals": s_refusals,
             "soak": s_soak}

if __name__ == "__main__":
    if sys.argv[1:2] == ["soak-seeds"]:               # python tests/emu/restart_scenarios.py soak-seeds <first> <count> [cases]
        for seed in range(int(sys.argv[2]), int(sys.argv[2]) + int(sys.argv[3])):
            soak(seed, int(sys.argv[4]) if len(sys.argv) > 4 else 12)
            print("ok soak seed", seed, flush=True)
        sys.exit(0)
    for name in (sys.argv[1:] or list(SCENARIOS)):
        SCENARIOS[name]()
        print("ok", name, flush=True)
