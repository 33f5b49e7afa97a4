"""Push programs of the streaming sessions: fade_in / fade_out / linear_gain_ramp / take_duration / distortion (with AMPLIFY and SPEED
among them) at the front of a source's chain, applied as the PCM is pushed (k_fifo_scatter<true>), and rb_session_push_silence for
Player::pause.  Every scenario compares the session's output bit for bit with the oracle's literal chains summed in the documented
slot order (tests/emu/layout_scenarios.py), and within 1e-5 * peak with the oracle's sequential mixer.

    python tests/emu/front_fx_scenarios.py <scenario> ...
runs them on the host-emulated library; tests/test_session_front_fx.py runs them there and on the device."""
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
import layout_scenarios as L                          # noqa: E402
import oracle                                         # noqa: E402
import rodio_b200 as rb                               # noqa: E402
from rodio_b200 import _capi as capi                  # noqa: E402
from helpers import assert_bit_exact, assert_close_peak, noise, to_oracle   # noqa: E402

MS = 1_000_000
HELD = capi.RB_SESSION_HELD


def take_ns(rate, ci, approx_ms, whole=True):
    """A duration near approx_ms whose take lets through a whole number of frames (whole) or ends inside a frame."""
    dps = 10**9 // (rate * ci)
    ns = approx_ms * MS
    while ((ns // dps) % ci == 0) != whole:
        ns += dps
    return ns


def apply_prog(s, prog):
    for op in prog:
        k = op[0]
        s = {"fade_in": lambda: s.fade_in(op[1]), "fade_out": lambda: s.fade_out(op[1]), "amp": lambda: s.amplify(op[1]),
             "speed": lambda: s.speed(op[1]), "dist": lambda: s.distortion(op[1], op[2]),
             "ramp": lambda: s.linear_gain_ramp(op[1], op[2], op[3], op[4]), "take": lambda: s.take_duration(op[1], op[2])}[k]()
    return s


class FSrc(L.Src):
    """A layout source (chain variant `kind`) whose chain begins with the push program `prog` (tuples, see apply_prog)."""

    def __init__(self, ci, rate, prog=(), **kw):
        super().__init__(ci, rate, **kw)
        self.prog = list(prog)

    def chain(self, mix_ch, mix_rate, pcm=None, pre=None, pauses=()):
        pcm = np.zeros(0, np.float32) if pcm is None else pcm
        s = apply_prog(rb.TestSource(pcm, self.ci, self.rate), self.prog)
        if pauses:                                    # Pausable behind the program: Player::pause / play at known positions
            s = s.speed(1.0)
            shift = 0
            for at, frames in pauses:
                s = s.pause_at(at + shift, frames)
                shift += frames * self.ci
        pre = self.pre if pre is None else pre
        if self.kind == "front":
            s = s.amplify(pre).low_pass(self.lp).amplify(self.mid)
            s = rb.UniformSourceIterator(s, mix_ch, mix_rate)
            return s.amplify(self.gain) if self.gain is not None else s
        if self.kind == "pre":
            s = s.amplify(pre)
        if self.kind == "speed":
            s = s.speed(self.speed)
        s = rb.UniformSourceIterator(s, mix_ch, mix_rate)
        if self.lp:
            s = s.low_pass(self.lp)
        return s.amplify(self.gain) if self.gain is not None else s

    def eff_rate(self):
        r = self.rate
        for op in self.prog:
            if op[0] == "speed":
                r = capi.lib().rb_speed_sample_rate(r, op[1])
        return capi.lib().rb_speed_sample_rate(r, self.speed) if self.kind == "speed" else r


def per_source(real, mix_ch, mix_rate):
    """The oracle's stream of each chain, a last partial frame (a take that ends inside a frame) completed with 0.0 as the
    session's padding: +0.0 added to the mix changes nothing there."""
    out = []
    for x in real:
        y = oracle.chain_uniform(to_oracle(x), mix_ch, mix_rate)
        if y.size % mix_ch:
            y = np.concatenate([y, np.zeros(mix_ch - y.size % mix_ch, np.float32)])
        out.append(y)
    return out


def check(got, srcs, real, starts, mix_ch, mix_rate, what):
    per = per_source(real, mix_ch, mix_rate)
    want = L.slot_expected(per, starts, srcs, mix_ch, mix_rate)
    assert_bit_exact(got, want[:got.size], what)
    assert got.size == want.size or not np.any(want[got.size:]), what + ": tail"
    ref = oracle.mixer([to_oracle(x, st * mix_ch) for x, st in zip(real, starts)], mix_ch, mix_rate)
    n = min(got.size, ref.size)
    assert_close_peak(got[:n], ref[:n], 1e-5, what + ": vs the sequential mixer")
    return want


def run(srcs, mix_ch, mix_rate, seed, what, packed=True, block=480, hand_over=None, split=True):
    rng = np.random.default_rng(seed)
    hooks = None
    if hand_over is not None:
        def swap(sess, _):
            t = L.session(srcs, mix_ch, mix_rate, block=block)
            t.set_state(sess.get_state())
            sess.close()
            return t
        hooks = {hand_over: swap}
    sess = L.session(srcs, mix_ch, mix_rate, block=block)
    got, sess = L.drive(sess, srcs, rng, [max(1, s.rate // 150) for s in srcs], block, packed=packed, hooks=hooks, split=split)
    sess.close()
    real = [s.chain(mix_ch, mix_rate, s.pcm) for s in srcs]
    return check(got, srcs, real, [s.start for s in srcs], mix_ch, mix_rate, what)


# ---------------------------------------------------------------------------------------------------------------------
def s_adapters():
    """fade_in, fade_out, linear_gain_ramp with and without clamp_end, distortion, take_duration with and without the fade-out
    filter, up-sampling, same-rate and down-sampling sources, in a stereo and a 6-channel mixer; random splits, a hand-over in
    the middle of the ramps and takes."""
    for mix_ch, cis, packed in ((2, (2, 1, 2, 2), True), (6, (6, 2, 3, 1), False)):
        srcs = []
        for k, rate in enumerate((44100, 48000, 96000, 22050)):
            ci = cis[k % len(cis)]
            progs = [[("fade_in", 9 * MS)], [("fade_out", 11 * MS)], [("ramp", 7 * MS, 0.2, 1.7, True)], [("ramp", 13 * MS, 1.5, 0.1, False)],
                     [("dist", 3.0, 0.5)], [("take", take_ns(rate, ci, 14), False)], [("take", take_ns(rate, ci, 12), True)],
                     [("fade_in", 5 * MS), ("take", take_ns(rate, ci, 15), True)]]
            for j, prog in enumerate(progs):
                srcs.append(FSrc(ci, rate, prog, lp=700 if j % 2 else None, gain=0.8 if j % 3 else None, frames=rate // 50 + 7 * j,
                                 start=0 if j % 3 else 11 * j, seed=100 * k + j))
        run(srcs, mix_ch, 48000, 3 + mix_ch, f"adapters, {mix_ch}-channel mixer", packed=packed, hand_over=2, block=400)


def s_mid_frame_takes():
    """Takes that end inside a frame (padding) for 1-, 2-, 3- and 6-channel sources at the mixer's rate, with and without the
    fade-out filter, ramps and distortion behind the take (they see its padding), amplify behind the conversion; and a long take
    (more than 32768 samples) at the mixer's rate."""
    srcs = []
    for k, ci in enumerate((1, 2, 3, 6) * 2):
        fade = k >= 4
        prog = [("take", take_ns(48000, ci, 9 + k, whole=(ci == 1)), fade), ("fade_out", 4 * MS), ("dist", 2.0, 0.7)] if k % 2 else \
               [("fade_in", 3 * MS), ("take", take_ns(48000, ci, 10 + k, whole=(ci == 1)), fade)]
        srcs.append(FSrc(ci, 48000, prog, lp=None, gain=0.9, frames=800 + 13 * k, start=5 * k, seed=300 + k))
    srcs.append(FSrc(2, 48000, [("fade_in", 200 * MS), ("take", 400 * MS, True)], lp=500, frames=21000, seed=399))
    run(srcs, 6, 48000, 9, "mid-frame takes", hand_over=3, block=512)


def s_program_variants():
    """Programs with AMPLIFY and SPEED between the adapters, combined with a filter in front, a filter behind, a gain in front (the
    Player's volume) and speed in front of the conversion."""
    srcs = []
    for k, kind in enumerate(("behind", "front", "pre", "speed") * 2):
        ci, rate = (2, 1, 6, 3)[k % 4], (44100, 32000, 48000, 24000)[k // 2 % 4]
        eff = capi.lib().rb_speed_sample_rate(rate, 1.25)
        prog = [("amp", 0.7), ("fade_in", 6 * MS), ("speed", 1.25), ("dist", 1.8, 0.6), ("amp", 1.3),
                ("take", take_ns(eff, ci, 13), bool(k % 2)), ("speed", 0.8)]
        if k >= 4:
            prog = prog[::-1][1:] + [("ramp", 5 * MS, 1.0, 0.3, True)]
        srcs.append(FSrc(ci, rate, prog, kind=kind, pre=(0.9, 0.6, -0.5, 1.1)[k % 4], frames=700 + 21 * k, start=0 if k % 2 else 17 * k,
                         seed=400 + k))
    run(srcs, 6, 48000, 13, "program variants", hand_over=2)


def s_split_invariance():
    """1- to 7-frame pushes, single and packed, random renders: the bytes of a one-block render."""
    srcs = [FSrc(ci, r, prog, lp=lp, frames=500 + 9 * k, seed=500 + k) for k, (ci, r, prog, lp) in enumerate([
        (6, 48000, [("fade_in", 6 * MS), ("take", take_ns(48000, 6, 8, whole=False), True)], None),
        (2, 44100, [("ramp", 5 * MS, 0.0, 2.0, False), ("dist", 1.5, 0.8)], 700),
        (1, 22050, [("take", take_ns(22050, 1, 15), False), ("fade_out", 9 * MS)], 700),
        (3, 96000, [("speed", 1.1), ("fade_in", 3 * MS)], 700),
        (2, 48000, [], 700)])]
    sess = L.session(srcs, 6, 48000, block=8192)
    for i, s in enumerate(srcs):
        sess.push(i, s.pcm, end_of_stream=True)
    whole, done = [], False
    while not done:
        block, done = sess.render(8192)
        whole.append(block)
    whole = np.concatenate(whole)
    sess.close()
    check(whole, srcs, [s.chain(6, 48000, s.pcm) for s in srcs], [0] * len(srcs), 6, 48000, "one-block render")
    rng = np.random.default_rng(5)
    for packed in (True, False):
        sess = L.session(srcs, 6, 48000, block=512)
        pos, got, done = [0] * len(srcs), [], False
        while not done:
            blocks, eos = [], []
            for i, s in enumerate(srcs):
                total = s.pcm.size // s.ci
                k = min(int(rng.integers(1, 8)), total - pos[i])
                blocks.append(s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)])
                pos[i] += k
                eos.append(pos[i] == total)
            if packed:
                sess.push_packed(blocks, eos)
            else:
                for i, (b, e) in enumerate(zip(blocks, eos)):
                    sess.push(i, b, end_of_stream=e)
            block, done = sess.render(int(rng.integers(1, 12)))
            got.append(block)
        sess.close()
        got = np.concatenate(got)
        assert np.array_equal(got.view(np.uint32), whole.view(np.uint32)), f"split (packed={packed}) differs from the one-block render"


def s_controls():
    """set_volume and set_amplify on program sources, skip of one, a held source queued behind a take (it starts on the frame
    after the take's padded last frame), pushes after the take has ended (accepted and dropped)."""
    mix_ch, mix_rate = 2, 48000
    srcs = [FSrc(2, 44100, [("fade_in", 4 * MS), ("take", take_ns(44100, 2, 30), True)], kind="pre", pre=1.0, frames=3000, seed=600),
            FSrc(1, 32000, [("fade_in", 8 * MS)], kind="pre", pre=1.0, frames=1500, seed=601),
            FSrc(2, 48000, [("take", take_ns(48000, 2, 21, whole=False), False)], kind="pre", pre=1.0, lp=None, frames=2500, seed=602),
            FSrc(2, 22050, [("dist", 2.5, 0.4)], kind="pre", pre=1.0, frames=4000, seed=603)]
    starts = [0, HELD, 0, 0]
    sess = L.session(srcs, mix_ch, mix_rate, starts=starts, block=256)
    sess.follow(1, 0)                                 # 1 plays behind 0's take
    sess.set_volume(2, 0.5)
    sess.set_amplify(3, 0.25)
    got, pos, marks = [], [0] * 4, {}
    for rnd in range(400):
        if rnd == 4:
            t = L.session(srcs, mix_ch, mix_rate, starts=starts, block=256)
            t.set_state(sess.get_state())
            sess.close()
            sess = t
        if rnd == 9:
            marks["T3"] = sum(b.size for b in got) // mix_ch
            sess.skip(3)
        blocks, eos = [], []
        for i, s in enumerate(srcs):
            total = s.pcm.size // s.ci
            k = 0 if (i == 3 and rnd >= 9) else min(s.rate // 100, total - pos[i])
            blocks.append(s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)])
            pos[i] += k
            eos.append(pos[i] == total and not (i == 3 and rnd >= 9))
        sess.push_packed(blocks, eos)                 # source 0's take ends long before its input: the rest is dropped
        ended = False
        while True:
            block, ended = sess.render(256)
            got.append(block)
            if block.size == 0 or ended:
                break
        if ended:
            break
    sess.push(0, srcs[0].pcm[:20])                    # after the take: RB_OK, dropped
    sess.close()
    got = np.concatenate(got)
    n3 = marks["T3"]
    g = math.gcd(22050, mix_rate)
    fpos = min(((n3 - 1) * (22050 // g)) // (mix_rate // g) + 2, pos[3])
    pcms = [s.pcm for s in srcs]
    pcms[3] = pcms[3][:2 * fpos]
    real = [s.chain(mix_ch, mix_rate, p, pre=(0.5 if i == 2 else None)) for i, (s, p) in enumerate(zip(srcs, pcms))]
    real[3] = rb.UniformSourceIterator(apply_prog(rb.TestSource(pcms[3], 2, 22050), srcs[3].prog).amplify(1.0), mix_ch, mix_rate).low_pass(
        srcs[3].lp).amplify(0.25)
    per = per_source(real, mix_ch, mix_rate)
    joined = [0, per[0].size // mix_ch, 0, 0]
    want = L.slot_expected(per, joined, srcs, mix_ch, mix_rate)
    assert_bit_exact(got, want[:got.size], "controls on program sources")
    assert got.size == want.size or not np.any(want[got.size:]), "tail"
    ref = oracle.mixer([to_oracle(x, st * mix_ch) for x, st in zip(real, joined)], mix_ch, mix_rate)
    assert_close_peak(got, ref[:got.size], 1e-5, "sequential mixer")


def pause_case(srcs, mix_ch, mix_rate, pauses, what, hand_over=None, block=300):
    """Drive with 10 ms pushes; pauses[i] = [(frames pushed before, silent frames), ...] pushed as silence at those points."""
    sess = L.session(srcs, mix_ch, mix_rate, block=block)
    pos, got, rnd, ended = [0] * len(srcs), [], 0, False
    todo = [list(p) for p in pauses]
    while not ended:
        if rnd == hand_over:
            t = L.session(srcs, mix_ch, mix_rate, block=block)
            t.set_state(sess.get_state())
            sess.close()
            sess = t
        for i, s in enumerate(srcs):
            total = s.pcm.size // s.ci
            k = min(s.rate // 100, total - pos[i])
            if todo[i] and pos[i] <= todo[i][0][0] < pos[i] + k + 1:
                at, n = todo[i].pop(0)
                sess.push(i, s.pcm[s.ci * pos[i]: s.ci * at])
                pos[i] = at
                sess.push_silence(i, n)
                continue
            sess.push(i, s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)], end_of_stream=(pos[i] + k == total and not todo[i]))
            pos[i] += k
        while True:
            b, ended = sess.render(block)
            got.append(b)
            if b.size == 0 or ended:
                break
        rnd += 1
        assert rnd < 10000
    sess.close()
    got = np.concatenate(got)
    real = [s.chain(mix_ch, mix_rate, s.pcm, pauses=[(at * s.ci, n) for at, n in p]) for s, p in zip(srcs, pauses)]
    check(got, srcs, real, [s.start for s in srcs], mix_ch, mix_rate, what)


def s_pause():
    """push_silence in the middle of a fade and of a take equals program.speed(1).pause_at(at, frames).amplify(v) (Pausable, RB_FX_PAUSE);
    a hand-over after a silence.  (Behind a take rodio's conversion counts the pause's zeros against the take and restarts early:
    the paused takes are at the mixer's rate, where a restart changes nothing; sessions refuse silence for the others.)"""
    srcs = [FSrc(2, 48000, [("fade_in", 40 * MS), ("take", take_ns(48000, 2, 120), True)], kind="pre", pre=0.8, lp=None, frames=6000, seed=700),
            FSrc(1, 48000, [("fade_out", 60 * MS)], kind="pre", pre=1.2, frames=4000, seed=701),
            FSrc(6, 48000, [("take", take_ns(48000, 6, 70, whole=False), True), ("dist", 1.2, 0.9)], kind="pre", pre=0.5, lp=None, frames=5000,
                 seed=702),
            FSrc(2, 96000, [("ramp", 30 * MS, 0.1, 1.0, False)], kind="pre", pre=1.0, frames=9000, seed=703)]
    pauses = [[(900, 700), (3000, 200)], [(1000, 480)], [(1500, 333)], [(2000, 1000)]]
    pause_case(srcs, 6, 48000, pauses, "pause mid-fade and mid-take", hand_over=12)


def s_large_pushes():
    """Pushes far larger than the FIFO into sources whose take cuts them, and again after the take has ended -- packed (next to a
    source fed in small blocks) and single: only what the take lets through is staged and kept, the rest is dropped with RB_OK."""
    mix_ch, mix_rate, fifo = 2, 48000, 64
    srcs = [FSrc(2, 48000, [("fade_in", MS // 2), ("take", take_ns(48000, 2, 1), True)], lp=None, frames=4000, seed=800),
            FSrc(1, 44100, [("fade_in", 20 * MS)], lp=700, frames=3000, seed=801),
            FSrc(6, 48000, [("take", take_ns(48000, 6, 1, whole=False), False), ("dist", 1.5, 0.6)], lp=None, frames=4000, seed=802)]
    for packed in (True, False):
        sess = L.session(srcs, mix_ch, mix_rate, block=64, fifo=fifo)
        pos1, got, ended, rnd = 0, [], False, 0
        while not ended:
            k = min(40, 3000 - pos1)
            blocks = [srcs[0].pcm, srcs[1].pcm[pos1:pos1 + k], srcs[2].pcm]   # the cut sources get their whole PCM every round
            pos1 += k
            if packed:
                sess.push_packed(blocks, [False, pos1 == 3000, False])
            else:
                for i, b in enumerate(blocks):
                    sess.push(i, b, end_of_stream=(i == 1 and pos1 == 3000))
            while True:
                b, ended = sess.render(64)
                got.append(b)
                if b.size == 0 or ended:
                    break
            rnd += 1
            assert rnd < 1000
        sess.close()
        got = np.concatenate(got)
        check(got, srcs, [s.chain(mix_ch, mix_rate, s.pcm) for s in srcs], [0, 0, 0], mix_ch, mix_rate, f"large pushes (packed={packed})")


def s_refusals():
    """What sessions do not serve, and the errors of the new calls; the blob sizes of sessions without a program are those of
    versions 5 and 6."""
    U, I, S = capi.RB_ERR_UNSUPPORTED, capi.RB_ERR_INVALID_ARGUMENT, capi.RB_ERR_STATE

    def refused(make, status=U):
        try:
            make().close()
        except capi.RodioB200Error as e:
            assert e.status == status, e
        else:
            raise AssertionError("accepted")
    z = np.zeros(0, np.float32)
    T = lambda ci=2, rate=44100: rb.TestSource(z, ci, rate)
    mk = lambda s, ch=2: rb.Session([rb.UniformSourceIterator(s, ch, 48000)], 48000, mixer_channels=ch)
    # the adapters behind a filter in front, behind the conversion
    for fx in (lambda s: s.fade_in(MS), lambda s: s.take_duration(MS), lambda s: s.distortion(2, 1)):
        refused(lambda: mk(fx(T().low_pass(300))))
        refused(lambda: rb.Session([fx(rb.UniformSourceIterator(T(), 2, 48000))], 48000, mixer_channels=2))
    # the other adapters, in front of the conversion
    for fx in (lambda s: s.delay(MS), lambda s: s.reverb(MS, 0.5), lambda s: s.automatic_gain_control(), lambda s: s.limit(),
               lambda s: rb.Source._with(s, rb.Effect.make(capi.RB_FX_CHANNEL_VOLUME, u32=[2], f32=[0.5, 0.5])),
               lambda s: rb.Source._with(s, rb.Effect.make(capi.RB_FX_SPATIAL, f32=[0.0] * 9)),
               lambda s: s.mix(T()), lambda s: s.pause_at(10, 10)):
        refused(lambda: mk(fx(T()).fade_in(MS)))
        refused(lambda: mk(fx(T().fade_in(MS))))
    # invalid parameters: the batch planner's status
    refused(lambda: mk(rb.Source._with(T(), rb.Effect.make(capi.RB_FX_LINEAR_RAMP, u32=[0], f32=[0.0, 1.0], ns=[0]))), I)
    refused(lambda: mk(T().distortion(1.0, -0.5)), I)
    refused(lambda: mk(T(2, 600_000_000).take_duration(MS)), I)             # 1e9 / (rate * 2) == 0 ns per sample
    # takes rodio converts in restarts the session cannot follow, and padding a filter would see
    refused(lambda: mk(T(2, 44100).take_duration(take_ns(44100, 2, 1000))))  # 88200 samples, resampled
    refused(lambda: mk(T(2, 44100).take_duration(take_ns(44100, 2, 20, whole=False))))
    refused(lambda: mk(T(3, 48000).take_duration(take_ns(48000, 3, 1000)), 2))   # restarts inside a frame while dropping a channel
    refused(lambda: rb.Session([rb.UniformSourceIterator(T(2, 48000).take_duration(take_ns(48000, 2, 20, whole=False)), 2, 48000).low_pass(300)],
                               48000, mixer_channels=2))
    refused(lambda: mk(T(2, 48000).take_duration(take_ns(48000, 2, 20, whole=False)).amplify(float("inf"))))
    mk(T(2, 48000).take_duration(take_ns(48000, 2, 1000))).close()            # long takes at the mixer's rate are served
    mk(T(2, 44100).take_duration(take_ns(44100, 2, 300))).close()             # one run of whole frames: any rate
    # push_silence: a filter in front; silence that does not fit; after end_of_stream; set_volume on a program AMPLIFY only
    with rb.Session([rb.UniformSourceIterator(T().fade_in(MS).amplify(0.5).low_pass(300), 2, 48000),
                     rb.UniformSourceIterator(T().amplify(0.5).fade_in(MS), 2, 48000),
                     rb.UniformSourceIterator(T().fade_in(MS).amplify(0.5), 2, 48000)], 48000, fifo_frames=64, mixer_channels=2) as s:
        for call, status in ((lambda: s.push_silence(0, 4), U), (lambda: s.push_silence(1, 65), capi.RB_ERR_BUFFER_TOO_SMALL),
                             (lambda: s.set_volume(1, 0.3), S)):
            try:
                call()
            except capi.RodioB200Error as e:
                assert e.status == status, e
            else:
                raise AssertionError("accepted")
        s.set_volume(2, 0.3)
        with mk(T(2, 44100).take_duration(take_ns(44100, 2, 300))) as t:
            try:
                t.push_silence(0, 4)
            except capi.RodioB200Error as e:
                assert e.status == U
            else:
                raise AssertionError("silence behind a resampled take was accepted")
        s.push_silence(1, 64)
        s.push(2, noise(20, 1), end_of_stream=True)
        try:
            s.push_silence(2, 1)
        except capi.RodioB200Error as e:
            assert e.status == S
        else:
            raise AssertionError("silence after end_of_stream was accepted")
        blob = s.get_state()
        assert int.from_bytes(blob[4:8], "little") == 7
    # a blob whose programs differ
    a = rb.Session([rb.UniformSourceIterator(T().fade_in(MS), 2, 48000)], 48000, mixer_channels=2)
    b = rb.Session([rb.UniformSourceIterator(T().fade_in(2 * MS), 2, 48000)], 48000, mixer_channels=2)
    c = rb.Session([rb.UniformSourceIterator(T(), 2, 48000)], 48000, mixer_channels=2)
    for x, y in ((a, b), (a, c), (c, a)):
        try:
            y.set_state(x.get_state())
        except capi.RodioB200Error as e:
            assert e.status == I
        else:
            raise AssertionError("a blob with other programs was accepted")
    for x in (a, b, c):
        x.close()
    # sessions without a program: versions 5 and 6, sizes unchanged
    with L.session([L.Src(2, 44100, frames=500, seed=1), L.Src(1, 44100, frames=500, seed=2)], 2, 48000) as s:
        blob = s.get_state()
        assert int.from_bytes(blob[4:8], "little") == 5 and len(blob) == 32 + 112 * 2
    with L.session([L.Src(6, 44100, frames=500, seed=3), L.Src(2, 44100, frames=500, seed=4)], 6, 48000) as s:
        blob = s.get_state()
        assert int.from_bytes(blob[4:8], "little") == 6 and len(blob) == 32 + (112 + 8) * 4


SCENARIOS = {"adapters": s_adapters, "mid_frame_takes": s_mid_frame_takes, "program_variants": s_program_variants,
             "split_invariance": s_split_invariance, "controls": s_controls, "pause": s_pause, "large_pushes": s_large_pushes,
             "refusals": s_refusals}

if __name__ == "__main__":
    for name in (sys.argv[1:] or list(SCENARIOS)):
        SCENARIOS[name]()
        print("ok", name, flush=True)
