"""Span reports that change while a source plays (rb_session_push_spans / rb_session_push_packed_spans): a decoder reports the
length of the packet it decoded last (src/decoder/symphonia.rs:199-201), and the mixer's UniformSourceIterator asks at every
bootstrap before it pulls (src/source/uniform.rs:50-68), so a bootstrap on a packet boundary is told the previous packet's length.
The pushes carry the changes as marks.  Every scenario compares the session's output bit for bit with the oracle's literal chains
-- over a source that reports by the same marks (tests/emu/marked_oracle.py) -- summed in the documented slot order, and within 1e-5 * peak with the
oracle's sequential mixer; rb_session_source_runs must equal the bootstraps the oracle's iterator makes.

    python tests/emu/packet_scenarios.py <scenario> ...
runs them on the host-emulated library; tests/test_session_packets.py runs them there and on the device."""
import ctypes
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
import marked_oracle as M                             # noqa: E402
import oracle                                         # noqa: E402
import restart_scenarios as R                         # noqa: E402
import rodio_b200 as rb                               # noqa: E402
from rodio_b200 import _capi as capi                  # noqa: E402
from helpers import assert_bit_exact, assert_close_peak, to_oracle   # noqa: E402

F, L = R.F, R.L
CAP = R.CAP
VARIANTS = R.VARIANTS


def symphonia_marks(packets):
    """Span marks of a decoder whose packets hold packets[k] samples, by symphonia's rule: current_span_len() is the length of
    the packet that holds the last sample yielded, packet 0 before any pull (the constructor decodes it, symphonia.rs:173-179;
    next() decodes the following one when it finds the buffer exhausted, :344-411).  Returns (report before the first pull,
    [(samples yielded, report), ...]) with absolute positions; a mark only where the report changes."""
    marks, start, cur = [], 0, packets[0]
    for k, n in enumerate(packets):
        if k and n != cur:
            marks.append((start + 1, n))         # the first sample of packet k has been yielded
        cur = n if k else cur
        start += n
    return packets[0], marks


def report_at(initial, marks, p):
    """The report after p samples have been yielded: the last mark at or before p."""
    r = initial
    for at, span in marks:
        if at > p:
            break
        r = span
    return r


def bootstraps(total, ci, initial, marks, pauses=(), take=None):
    """Converter runs UniformSourceIterator makes over a source of `total` samples that reports by `marks`, with pauses (frame,
    frames) of zeros behind it (counted against the run, not yielded by the source) and a take of `take` samples: the runs that
    produce an output."""
    segs, p = [], 0                             # the chain's samples: ('real', n) / ('zero', n)
    end = total if take is None else min(total, take)
    for at, n in sorted(pauses):
        at = min(at * ci, end)
        if at > p:
            segs.append(["real", at - p])
        segs.append(["zero", n * ci])
        p = at
    if end > p:
        segs.append(["real", end - p])
    runs, p = 0, 0
    while segs:
        rep = report_at(initial, marks, p)
        left = None if take is None else take - p
        n = rep if rep else None
        n = min(n, CAP) if n is not None else None
        if left is not None:
            n = min(n, left) if n is not None else min(left, CAP)
        runs += 1
        if n is None:
            break
        while n and segs:
            k = min(n, segs[0][1])
            if segs[0][0] == "real":
                p += k
            segs[0][1] -= k
            n -= k
            if segs[0][1] == 0:
                segs.pop(0)
    return runs


def decoder_packets(rng, frames, ci, sizes=(64, 128, 256, 576, 1024), stretch=(1, 6)):
    """Packet sizes (samples) of a decoder: stretches of equal packets with switches between them, the last one short."""
    out, left = [], frames
    while left > 0:
        n = int(rng.choice(sizes))
        for _ in range(int(rng.integers(*stretch))):
            k = min(n, left)
            out.append(k * ci)
            left -= k
            if not left:
                break
    return out


class PSrc(R.RSrc):
    """A restart source whose base reports by marks: `initial` (samples, 0: None) before the first, then marks [(at, span)]."""

    def __init__(self, ci, rate, prog=(), packets=None, initial=None, marks=(), **kw):
        super().__init__(ci, rate, prog, **kw)
        if packets is not None:
            initial, marks = symphonia_marks(packets)
        self.span = initial or 0
        self.marks = [(int(a), int(s)) for a, s in marks]

    def take_samples(self):
        for op in self.prog:
            if op[0] == "take":
                return (op[1] // (10**9 // (self.rate * self.ci)))
        return None

    def runs(self, pauses=(), upto=None):
        if self.rate == MIX_RATE[0]:
            return None
        n = self.pcm.size if upto is None else upto * self.ci
        return bootstraps(n, self.ci, self.span, self.marks, pauses, self.take_samples())

    def push_marks(self, a, b):
        """The marks of a push of samples [a, b): relative to a, a change after the push's last sample goes to the next push."""
        return [(at - a, s) for at, s in self.marks if a <= at < b]


MIX_RATE = [48000]
BLOBS = []   # versions of the state blobs handed over


def chain_o(x, s, mix_ch, mix_rate):
    """The oracle's stream of chain x over source s, its base reporting by s's marks."""
    return M.chain_uniform(to_oracle(x), s.marks, mix_ch, mix_rate)


def check(got, srcs, real, starts, mix_ch, mix_rate, what):
    per = []
    for x, s in zip(real, srcs):
        y = chain_o(x, s, mix_ch, mix_rate)
        if y.size % mix_ch:
            y = np.concatenate([y, np.zeros(mix_ch - y.size % mix_ch, np.float32)])
        per.append(y)
    want = L.slot_expected(per, starts, srcs, mix_ch, mix_rate)
    assert_bit_exact(got, want[:got.size], what)
    assert got.size == want.size or not np.any(want[got.size:]), what + ": tail"
    ref = M.mixer([to_oracle(x, st * mix_ch) for x, st in zip(real, starts)], [s.marks for s in srcs], mix_ch, mix_rate)
    n = min(got.size, ref.size)
    assert_close_peak(got[:n], ref[:n], 1e-5, what + ": vs the sequential mixer")
    return want


def session(srcs, mix_ch, mix_rate, starts=None, fifo=4096, block=480):
    return R.session(srcs, mix_ch, mix_rate, starts=starts, fifo=fifo, block=block)


def drive(sess, srcs, rng=None, push=None, block=480, pauses=None, hooks=None, packed=True, per_render=None):
    """R.drive with each push's marks; per_render(sess, launches this render) after every render."""
    push = push or [max(1, s.rate // 100) for s in srcs]
    pos, got, ended, rnd = [0] * len(srcs), [], False, 0
    todo = [list(p) for p in (pauses or [[]] * len(srcs))]
    while not ended:
        if hooks and rnd in hooks:
            r = hooks[rnd](sess, sum(b.size for b in got) // sess.channels)
            sess = r if r is not None else sess
        blocks, eos, silence, spans = [], [], [], []
        for i, s in enumerate(srcs):
            k = min(int(rng.integers(0, 2 * push[i] + 1)) if rng is not None else push[i], s.frames() - pos[i])
            if todo[i] and pos[i] <= todo[i][0][0] <= pos[i] + k:
                k = todo[i][0][0] - pos[i]
                silence.append((i, todo[i].pop(0)[1]))
            blocks.append(s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)])
            spans.append(s.push_marks(s.ci * pos[i], s.ci * (pos[i] + k)))
            pos[i] += k
            eos.append(pos[i] == s.frames() and not todo[i])
        if packed:
            sess.push_packed(blocks, eos, spans=spans)
        else:
            for i, (b, e) in enumerate(zip(blocks, eos)):
                if b.size or e:
                    sess.push(i, b, end_of_stream=e, spans=spans[i])
        for i, n in silence:
            sess.push_silence(i, n)
        while True:
            l0 = sess.restart_launches()
            b, ended = sess.render(int(rng.integers(1, block + 1)) if rng is not None else block)
            if per_render:
                per_render(sess, sess.restart_launches() - l0)
            got.append(b)
            if b.size == 0 or ended:
                break
        rnd += 1
        assert rnd < 200000
    return np.concatenate(got), sess


def hand_over(srcs, mix_ch, mix_rate, **kw):
    def swap(sess, _):
        blob = sess.get_state()
        BLOBS.append(int.from_bytes(blob[4:8], "little"))
        t = session(srcs, mix_ch, mix_rate, **kw)
        t.set_state(blob)
        sess.close()
        return t
    return swap


def run(srcs, mix_ch, mix_rate, seed, what, block=480, swap_at=None, pauses=None, fifo=4096, packed=True, split=True, per_render=None):
    MIX_RATE[0] = mix_rate
    sess = session(srcs, mix_ch, mix_rate, block=block, fifo=fifo)
    hooks = {swap_at: hand_over(srcs, mix_ch, mix_rate, block=block, fifo=fifo)} if swap_at is not None else None
    got, sess = drive(sess, srcs, np.random.default_rng(seed) if split else None, block=block, pauses=pauses, hooks=hooks, packed=packed,
                      per_render=per_render)
    runs = [sess.source_runs(i) for i in range(len(srcs))]
    sess.close()
    real = [s.chain(mix_ch, mix_rate, s.pcm, pauses=[(at * s.ci, n) for at, n in (pauses[i] if pauses else [])]) for i, s in enumerate(srcs)]
    check(got, srcs, real, [s.start for s in srcs], mix_ch, mix_rate, what)
    for i, s in enumerate(srcs):
        want = s.runs(pauses[i] if pauses else ())
        assert want is None or runs[i] == want, (what, i, runs[i], want)
    return runs


# ---------------------------------------------------------------------------------------------------------------------
def s_symphonia_rule():
    """The helper, by hand: packets of 3, 5, 2 and 40000 samples (mono).  Before any pull the report is 3; it becomes 5 once
    the first sample of packet 1 (sample 3) is yielded, 2 at sample 8, 40000 at sample 10.  The literal iterator bootstraps at 0
    (report 3: run [0, 3)), at 3 (still 3, the lag: run [3, 6), across the boundary), at 6 (5: [6, 11)), at 11 (40000, capped:
    [11, 32779)) and at 32779 (40000 again -- the whole buffer, though the bootstrap is in mid-packet: the rest)."""
    initial, marks = symphonia_marks([3, 5, 2, 40000])
    assert (initial, marks) == (3, [(4, 5), (9, 2), (11, 40000)]), (initial, marks)
    assert [report_at(initial, marks, p) for p in (0, 3, 4, 6, 8, 9, 10, 11, 32779)] == [3, 3, 5, 5, 5, 2, 2, 40000, 40000]
    total = 40010
    assert bootstraps(total, 1, initial, marks) == 5
    # the oracle's UniformSourceIterator over the marked source (tests/emu/marked_oracle.cpp): a run emits its last frame raw, so a ramp shows where runs end
    pcm = np.arange(total, dtype=np.float32)
    y = M.chain_uniform(oracle.Stream(pcm, 1, 44100, [], span_len=initial), marks, 1, 88200)
    # at 1:2 a run of L frames gives 2 L - 1 outputs: every output interpolates except the last, which is the raw last frame
    lens = [3, 3, 5, 32768, total - 32779]
    assert y.size == sum(2 * n - 1 for n in lens), y.size
    o = 0
    for a, n in zip(np.cumsum([0] + lens[:-1]), lens):
        seg = y[o:o + 2 * n - 1]
        assert seg[0] == a and seg[-1] == a + n - 1 and seg[-2] == a + n - 1.5, (a, n, seg[:3], seg[-3:])
        o += 2 * n - 1


def s_decoder():
    """Decoder-like packets (64 to 1024 frames in stretches, symphonia's lagged report) for mono, stereo, 4- and 8-channel sources
    in 2-, 6- and 8-channel mixers; up-, same- and down-sampling; all six chain variants; random unaligned pushes, single and
    packed; a hand-over in mid-stream."""
    BLOBS.clear()
    for m, mix_ch in enumerate((2, 6, 8)):
        rng = np.random.default_rng(70 + m)
        srcs = []
        for k, (ci, rate, frames) in enumerate([(2, 44100, 6000), (1, 44100, 5000), (2, 96000, 7000), (2, 48000, 3000), (4, 44100, 3000),
                                                (8, 22050, 2000), (1, 32000, 4000), (2, 88200, 5000)]):
            if ci > mix_ch and m == 0 and ci == 8:
                ci = 2
            srcs.append(PSrc(ci, rate, packets=decoder_packets(rng, frames, ci), frames=frames, start=0 if k % 3 else 5 * k,
                             seed=7000 + 100 * m + k, **VARIANTS[(k + m) % len(VARIANTS)]))
        run(srcs, mix_ch, 48000, 31 + m, f"decoder packets, {mix_ch}-channel mixer", swap_at=4, block=333 if m else 480, fifo=8192,
            packed=bool(m != 1))
    assert BLOBS == [9, 9, 9], BLOBS


def s_reports():
    """A report that goes to None and back (a bootstrap under None: one run for the rest), reports above 32768, and a constant
    report given by marks -- bit-identical to a session declared with that span_len."""
    srcs = [PSrc(2, 44100, initial=2 * 300, marks=[(2 * 700, 0), (2 * 1500, 2 * 200)], frames=4000, seed=8000, **VARIANTS[2]),
            PSrc(2, 44100, initial=2 * 300, marks=[(2 * 700 + 1, 0), (2 * 800, 2 * 100)], frames=3000, seed=8001, **VARIANTS[0]),
            PSrc(1, 44100, initial=0, marks=[(0, 500), (3000, 0)], frames=6000, seed=8002, **VARIANTS[3]),
            PSrc(1, 22050, initial=40000, marks=[(33000, 70000), (34000, 100)], frames=40000, seed=8003, **VARIANTS[4]),
            PSrc(2, 96000, initial=0, marks=[(0, 2 * 20000), (2 * 17000, 2 * 30000)], frames=40000, seed=8004, **VARIANTS[1]),
            PSrc(1, 44100, initial=0, marks=[(1, 0)], frames=900, seed=8005, **VARIANTS[5])]
    runs = run(srcs, 2, 48000, 5, "reports: None and back, above 32768", swap_at=6, fifo=40000, block=480)
    assert runs[0] == 4 and runs[5] == 1, runs
    # constant report by marks vs the declared span_len, bit for bit
    a = PSrc(2, 44100, initial=0, marks=[(0, 512)], frames=3000, seed=8100, **VARIANTS[2])
    b = PSrc(2, 44100, initial=512, frames=3000, seed=8100, **VARIANTS[2])
    outs = []
    for s in (a, b):
        MIX_RATE[0] = 48000
        sess = session([s], 2, 48000)
        got, sess = drive(sess, [s], np.random.default_rng(9))
        outs.append(got)
        assert sess.source_runs(0) == -(-3000 // 256)
        sess.close()
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), "constant report by marks differs from span_len"


def s_many_cuts():
    """Runs of 2 to 40 frames: every render makes at most one RESTART launch per class, and the output matches the oracle."""
    rng = np.random.default_rng(11)
    srcs = []
    for k, (ci, rate) in enumerate([(2, 44100), (1, 44100), (2, 96000), (1, 22050), (2, 32000), (1, 96000)]):
        pk = [ci * int(rng.integers(2, 41)) for _ in range(200)]
        srcs.append(PSrc(ci, rate, packets=pk, frames=sum(pk) // ci, seed=9000 + k, **VARIANTS[k % len(VARIANTS)]))
    n_classes = len(L.slot_classes(srcs, 2, 48000))
    worst = [0]

    def per_render(sess, launches):
        worst[0] = max(worst[0], launches)
        assert launches <= n_classes, launches
    run(srcs, 2, 48000, 12, "runs of 2 to 40 frames", block=480, per_render=per_render)
    assert worst[0] > 0


def s_programs():
    """fade_in, take_duration with its fade-out filter and distortion in front of decoder packets; pauses counted against the run
    (placed off the marks: a change seen at the end of a push is delivered with the next push, after the silence)."""
    rng = np.random.default_rng(13)
    srcs, pauses = [], []
    for k in range(6):
        ci, frames = (2, 9000) if k % 2 else (1, 7000)
        take = ci * (frames - 1500 + 97 * k)
        prog = [("fade_in", 50 * R.MS), R.take_of(44100, ci, take), ("dist", 1.5, 0.7)] if k % 3 else [("fade_in", 50 * R.MS), R.take_of(44100, ci, take)]
        s = PSrc(ci, 44100, prog, packets=decoder_packets(rng, frames, ci), frames=frames, kind="pre", pre=1.0, lp=None if k % 2 else 700,
                 seed=9500 + k)
        p = []
        if k % 3 != 2:
            at = 1000 + 611 * k
            while any(m == at * ci for m, _ in s.marks):
                at += 1
            p = [(at, 300 + 50 * k)]
        srcs.append(s)
        pauses.append(p)
    run(srcs, 2, 48000, 14, "push programs with pauses", pauses=pauses, split=False, swap_at=9, fifo=8192)


def s_controls():
    """set_volume before and after a cut, a source queued behind one with packets (follow), skip inside a run."""
    mix_ch, mix_rate = 2, 48000
    rng = np.random.default_rng(15)
    srcs = [PSrc(2, 44100, packets=decoder_packets(rng, 3000, 2, sizes=(64, 96, 200)), frames=3000, kind="pre", pre=1.0, lp=700, seed=9700),
            PSrc(1, 22050, packets=decoder_packets(rng, 900, 1, sizes=(64, 100)), frames=900, kind="pre", pre=1.0, seed=9701),
            PSrc(2, 44100, packets=decoder_packets(rng, 3000, 2, sizes=(128, 300)), frames=3000, kind="pre", pre=1.0, seed=9702)]
    starts = [0, R.HELD, 0]
    MIX_RATE[0] = mix_rate
    sess = session(srcs, mix_ch, mix_rate, starts=starts, block=100)
    sess.follow(1, 0)
    for i, s in enumerate(srcs):
        n = 2000 if i == 2 else s.frames()
        sess.push(i, s.pcm[:s.ci * n], end_of_stream=(i != 2), spans=s.push_marks(0, s.ci * n))
    got, n, ended, marks = [], 0, False, {}
    for upto, act in ((700, "vol"), (1300, "skip"), (None, None)):
        while not ended and (upto is None or n < upto):
            b, ended = sess.render(100 if upto is None else min(100, upto - n))
            got.append(b)
            n += b.size // mix_ch
            if b.size == 0:
                break
        marks[act] = n
        if act == "vol":
            sess.set_volume(0, 0.5)
        elif act == "skip":
            sess.skip(2)
    runs = [sess.source_runs(i) for i in range(3)]
    sess.close()
    got = np.concatenate(got)
    # the same controls replayed on the oracle: the volume applies to the frames the converter pulls after the change, the skipped
    # source ends with the last frame its converter pulled -- both found from the runs the oracle's iterator makes
    f, t = R.ratio(44100, mix_rate)

    def run_lens(s, upto):
        lens, p = [], 0
        while p < upto:
            rep = report_at(s.span, s.marks, p * s.ci)
            n = min(min(rep, CAP) // s.ci if rep else upto, upto - p)
            lens.append(n)
            p += n
        return lens
    p1 = R.pulled_after(run_lens(srcs[0], 3000), f, t, marks["vol"])
    vol = np.ones(3000, np.float32)
    vol[p1:] = 0.5
    p_skip = R.pulled_after(run_lens(srcs[2], 2000), f, t, marks["skip"])
    real = [srcs[0].chain(mix_ch, mix_rate, (srcs[0].pcm.reshape(-1, 2) * vol[:, None]).reshape(-1)), srcs[1].chain(mix_ch, mix_rate, srcs[1].pcm),
            srcs[2].chain(mix_ch, mix_rate, srcs[2].pcm[:2 * p_skip])]
    per = [chain_o(x, s, mix_ch, mix_rate) for x, s in zip(real, srcs)]
    want = L.slot_expected(per, [0, per[0].size // mix_ch, 0], srcs, mix_ch, mix_rate)
    assert_bit_exact(got, want[:got.size], "controls around cuts")
    assert got.size == want.size or not np.any(want[got.size:]), "tail"
    assert runs[0] == srcs[0].runs() and runs[1] == srcs[1].runs() and runs[2] == bootstraps(2 * p_skip, 2, srcs[2].span, srcs[2].marks), runs


def s_refusals():
    """Marks on a session without the flag (RB_ERR_STATE), malformed marks (RB_ERR_INVALID_ARGUMENT), a run that is not whole frames
    and one under two frames (RB_ERR_UNSUPPORTED, where a bootstrap meets them): a refused push leaves the output as if it had not
    been made.  A report no bootstrap sees is not refused; same-rate sources ignore marks."""
    S, U, I = capi.RB_ERR_STATE, capi.RB_ERR_UNSUPPORTED, capi.RB_ERR_INVALID_ARGUMENT
    MIX_RATE[0] = 48000
    s = PSrc(2, 44100, initial=2 * 100, frames=2000, seed=9900, **VARIANTS[2])

    def refused(call, status):
        try:
            call()
        except capi.RodioB200Error as e:
            assert e.status == status, (e.status, status)
        else:
            raise AssertionError("accepted")
    x = s.pcm[:2 * 500]
    plain = R.session([s], 2, 48000, restarts=False)
    refused(lambda: plain.push(0, x, spans=[(0, 200)]), S)
    refused(lambda: plain.push_packed([x], spans=[[(0, 200)]]), S)
    plain.close()
    a, b = session([s], 2, 48000), session([s], 2, 48000)
    for sess in (a, b):
        sess.push(0, x[:2 * 150], spans=[(3, 2 * 90)])
    for bad, st in (([(5, 200), (5, 300)], I), ([(7, 200), (3, 300)], I), ([(2 * 500, 200)], I), ([(2 * 10, 201)], U), ([(2 * 10, 2)], U),
                    ([(2 * 10, 3)], U)):
        refused(lambda: a.push(0, x[2 * 150:], spans=bad), st)
        refused(lambda: a.push_packed([x[2 * 150:]], spans=[bad]), st)
    marks = (capi.rb_span_mark * 1)(capi.rb_span_mark(0, 200, 1))    # pad_ != 0
    xs = np.ascontiguousarray(x[2 * 150:])
    assert capi.lib().rb_session_push_spans(a._h, 0, xs.ctypes.data_as(ctypes.c_void_p), xs.size // 2, marks, 1, 0) == I
    assert capi.lib().rb_session_push_spans(a._h, 0, xs.ctypes.data_as(ctypes.c_void_p), xs.size // 2, None, 1, 0) == I
    # a report of one frame that no bootstrap meets is accepted; the next bootstrap refuses it, silence included
    for sess in (a, b):
        sess.push(0, x[2 * 150:2 * 200], spans=[(2 * 40 + 1, 2)])
    refused(lambda: a.push(0, x[2 * 200:]), U)
    refused(lambda: a.push_silence(0, 500), U)
    for sess in (a, b):
        sess.push(0, x[2 * 200:], spans=[(0, 2 * 64)], end_of_stream=True)
    outs = []
    for sess in (a, b):
        got, done = [], False
        while not done:
            o, done = sess.render(480)
            got.append(o)
        outs.append(np.concatenate(got))
        sess.close()
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), "a refused push changed the session"
    # same-rate sources accept marks and ignore them; a session that never received marks writes the blob of before
    q = PSrc(2, 48000, initial=0, frames=500, seed=9901, **VARIANTS[1])
    with session([q], 2, 48000) as t:
        assert int.from_bytes(t.get_state()[4:8], "little") == 5
        t.push(0, q.pcm, spans=[(0, 3), (7, 1)], end_of_stream=True)
        assert int.from_bytes(t.get_state()[4:8], "little") == 9
        o, done = [], False
        while not done:
            b, done = t.render(480)
            o.append(b)
        o = np.concatenate(o)
    assert_bit_exact(o, oracle.chain_uniform(to_oracle(q.chain(2, 48000, q.pcm)), 2, 48000) + np.float32(0.0), "same-rate source with marks")
    # a version-9 blob does not load into a session without the flag
    with session([s], 2, 48000) as t:
        t.push(0, x, spans=[(0, 2 * 64)])
        blob = t.get_state()
    with R.session([s], 2, 48000, restarts=False) as t:
        refused(lambda: t.set_state(blob), I)


def soak(seed, cases):
    """Random decoders: packet sizes, rates, layouts, chain variants, takes with pauses, random splits and hand-overs."""
    rng = np.random.default_rng(seed)
    for case in range(cases):
        mix_ch = int(rng.choice([1, 2, 2, 6]))
        mix_rate = int(rng.choice([48000, 44100]))
        srcs, pauses = [], []
        for k in range(int(rng.integers(1, 8))):
            ci = 1 if mix_ch == 1 else int(rng.choice([1, 2, 2, 4]))
            rate = int(rng.choice([44100, 22050, 48000, 96000, 32000]))
            frames = int(rng.integers(1, 2500))
            sizes = [int(v) for v in rng.choice([2, 3, 17, 64, 100, 576, 1152, 2048], size=3)]
            v = dict(VARIANTS[int(rng.integers(len(VARIANTS)))])
            prog, p = [], []
            if rng.random() < 0.3 and v.get("kind") != "front":
                take = ci * int(rng.integers(2, frames + 2))
                fade = bool(rng.random() < 0.5) and take * 1000 >= 2 * rate * ci
                prog = [("fade_in", 3 * R.MS), R.take_of(rate, ci, take, fade)]
            s = PSrc(ci, rate, prog, packets=decoder_packets(rng, frames, ci, sizes=sizes, stretch=(1, 4)), frames=frames,
                     start=0 if rng.random() < 0.6 else int(rng.integers(0, 300)), seed=95000 + 100 * case + k + 7919 * seed, **v)
            if prog and rng.random() < 0.5:
                at = int(rng.integers(0, min(frames, take // ci)))
                if not any(m == at * ci for m, _ in s.marks):
                    p = [(at, int(rng.integers(1, 200)))]
            srcs.append(s)
            pauses.append(p)
        try:
            run(srcs, mix_ch, mix_rate, 1000 * seed + case, f"soak seed {seed} case {case}", block=int(rng.choice([7, 64, 480])), pauses=pauses,
                swap_at=int(rng.integers(0, 6)) if rng.random() < 0.5 else None, packed=bool(rng.random() < 0.5), fifo=4096)
        except Exception:
            print("soak seed", seed, "case", case, [(s.ci, s.rate, s.span, s.marks[:6], s.frames(), s.kind, s.lp, s.gain, s.prog, s.start) for s in srcs],
                  pauses, flush=True)
            raise


def s_soak():
    soak(1, 10)


def scale(n=1024, hand_over_at=60):
    """1024 stereo 44.1 kHz decoders (packets of 64 to 1024 frames) into a 48 kHz stereo mixer, 10 ms packed pushes and renders, one
    hand-over: bit for bit."""
    rng = np.random.default_rng(77)
    srcs = [PSrc(2, 44100, packets=decoder_packets(rng, 30000 - 7 * (k % 50), 2), frames=30000 - 7 * (k % 50), kind="pre", pre=1.0,
                 lp=None if k % 3 else 700, start=0 if k % 7 else 3 * k, seed=60000 + k) for k in range(n)]
    run(srcs, 2, 48000, 0, f"{n} stereo decoders", block=480, swap_at=hand_over_at, split=False, fifo=8192)


SCENARIOS = {"symphonia_rule": s_symphonia_rule, "decoder": s_decoder, "reports": s_reports, "many_cuts": s_many_cuts,
             "programs": s_programs, "controls": s_controls, "refusals": s_refusals, "soak": s_soak}

if __name__ == "__main__":
    if sys.argv[1:2] == ["soak-seeds"]:               # python tests/emu/packet_scenarios.py soak-seeds <first> <count> [cases]
        for seed in range(int(sys.argv[2]), int(sys.argv[2]) + int(sys.argv[3])):
            soak(seed, int(sys.argv[4]) if len(sys.argv) > 4 else 10)
            print("ok soak seed", seed, flush=True)
        sys.exit(0)
    for name in (sys.argv[1:] or list(SCENARIOS)):
        SCENARIOS[name]()
        print("ok", name, flush=True)
