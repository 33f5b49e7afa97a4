"""Session layouts beyond mono and stereo: mixers of 1 to 12 channels, sources of 1 to 12 channels each, served as slot rows of
at most two channels (rb_api.cu, rb_session).  Every scenario compares the session's output bit for bit with the oracle's literal
chains (UniformSourceIterator with the real ChannelCountConverter) summed in the documented slot order, and within 1e-5 * peak
with the oracle's sequential mixer.

The scenarios run on whatever library rodio_b200 loads: the GPU tests (tests/test_session_layouts.py) call them on the device;
    python tests/emu/layout_scenarios.py <scenario> ...
runs them on the host-emulated library (the real host code over the mock runtime, kernels on the SIMT emulator)."""
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
import oracle                                         # noqa: E402
import rodio_b200 as rb                               # noqa: E402
from rodio_b200 import _capi as capi                  # noqa: E402
from helpers import assert_bit_exact, assert_close_peak, lanes_tree_sum, noise, to_oracle   # noqa: E402

HELD = capi.RB_SESSION_HELD
CTX = {"ctx": None}       # the GPU tests set a context of their own


class Src:
    """One session source: channels, rate and chain variant.
    kind: 'behind' = conversion -> [low_pass] -> [amplify]; 'pre' = amplify in front of it as well; 'front' = amplify -> low_pass
    -> amplify (the Player's volume) in front of the conversion, amplify behind; 'speed' = speed in front, filter and gain behind."""

    def __init__(self, ci, rate, kind="behind", lp=700, gain=0.8, pre=0.9, mid=0.7, speed=1.1, start=0, frames=900, seed=0):
        self.ci, self.rate, self.kind, self.lp, self.gain, self.pre, self.mid, self.speed = ci, rate, kind, lp, gain, pre, mid, speed
        self.start, self.seed = start, seed
        self.pcm = noise(ci * frames, 12000 + seed, 0.8)

    def chain(self, mix_ch, mix_rate, pcm=None, pre=None):
        pcm = np.zeros(0, np.float32) if pcm is None else pcm
        s = rb.TestSource(pcm, self.ci, self.rate)
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
        if self.gain is not None:
            s = s.amplify(self.gain)
        return s

    def eff_rate(self):
        return capi.lib().rb_speed_sample_rate(self.rate, self.speed) if self.kind == "speed" else self.rate

    def key(self):   # the chain variant that splits classes: filter behind, gain in front, filter in front
        return (self.kind != "front" and bool(self.lp), self.kind == "pre", self.kind == "front")


def slot_rows(ci, mix_ch):
    """(ch0, w, ci) of a source's rows: mono into a wider mixer is one row on channels 0 and 1; otherwise pairs of the
    min(ci, mix_ch) channels it feeds, an odd last channel alone."""
    if ci == 1 and mix_ch >= 2:
        return [(0, 2, 1)]
    k = min(ci, mix_ch)
    return [(c0, min(2, k - c0), min(2, k - c0)) for c0 in range(0, k, 2)]


def slot_classes(srcs, mix_ch, mix_rate):
    """Rows of the sources in the caller's order, stably partitioned by (rate pair, chain variant, slot)."""
    keys, classes = [], []
    for i, s in enumerate(srcs):
        g = math.gcd(s.eff_rate(), mix_rate)
        for slot in slot_rows(s.ci, mix_ch):
            k = (s.eff_rate() // g, mix_rate // g, s.key(), slot)
            if k not in keys:
                keys.append(k)
                classes.append([])
            classes[keys.index(k)].append((i, slot))
    return classes


def slot_expected(per, starts, srcs, mix_ch, mix_rate):
    """The documented order: per class, groups of 32 rows summed with the lane tree; mixer channel j = +0.0, then every group
    whose slot covers j, in class order."""
    frames = max([st + y.size // mix_ch for st, y in zip(starts, per)] + [0])
    acc = np.zeros((frames, mix_ch), np.float32)
    for cls in slot_classes(srcs, mix_ch, mix_rate):
        ch0, w, _ = cls[0][1]
        for g in range(0, len(cls), 32):
            lanes = np.zeros((32, frames, w), np.float32)
            for l, (i, _) in enumerate(cls[g:g + 32]):
                y = per[i].reshape(-1, mix_ch)
                lanes[l, starts[i]:starts[i] + y.shape[0]] = y[:, ch0:ch0 + w]
            acc[:, ch0:ch0 + w] = acc[:, ch0:ch0 + w] + lanes_tree_sum(lanes)
    return acc.reshape(-1)


def session(srcs, mix_ch, mix_rate, starts=None, fifo=4096, block=480, master=()):
    return rb.Session([s.chain(mix_ch, mix_rate) for s in srcs], mix_rate, fifo_frames=fifo, max_block_frames=block,
                      mix_starts=starts if starts is not None else [s.start for s in srcs], ctx=CTX["ctx"], mixer_channels=mix_ch,
                      master=master)


def drive(sess, srcs, rng, push_frames, render_frames, packed=True, hooks=None, split=True):
    """Push up to push_frames[i] frames per source and round (random amounts when split), render until nothing comes."""
    pos, got, ended, rnd = [0] * len(srcs), [], False, 0
    while not ended:
        if hooks and rnd in hooks:
            r = hooks[rnd](sess, sum(b.size for b in got))
            sess = r if r is not None else sess
        blocks, eos = [], []
        for i, s in enumerate(srcs):
            total = s.pcm.size // s.ci
            k = int(rng.integers(0, 2 * push_frames[i] + 1)) if split else push_frames[i]
            k = min(k, total - pos[i])
            blocks.append(s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)])
            pos[i] += k
            eos.append(pos[i] == total)
        if packed:
            sess.push_packed(blocks, eos)
        else:
            for i, (b, e) in enumerate(zip(blocks, eos)):
                if b.size or e:
                    sess.push(i, b, end_of_stream=e)
        while True:
            n = int(rng.integers(1, render_frames + 1)) if split else render_frames
            block, ended = sess.render(n)
            got.append(block)
            if block.size == 0 or ended:
                break
        rnd += 1
        assert rnd < 100000
    return np.concatenate(got), sess


def check(got, srcs, mix_ch, mix_rate, starts, what, pcms=None):
    pcms = pcms or [s.pcm for s in srcs]
    real = [s.chain(mix_ch, mix_rate, p) for s, p in zip(srcs, pcms)]
    per = [oracle.chain_uniform(to_oracle(x), mix_ch, mix_rate) for x in real]
    want = slot_expected(per, starts, srcs, mix_ch, mix_rate)
    assert_bit_exact(got, want[:got.size], what)
    assert got.size == want.size or not np.any(want[got.size:]), what + ": tail"
    ref = oracle.mixer([to_oracle(x, st * mix_ch) for x, st in zip(real, starts)], mix_ch, mix_rate)   # mix_start in samples
    assert_close_peak(got, ref[:got.size], 1e-5, what + ": vs the sequential mixer")
    return want


def run_case(srcs, mix_ch, mix_rate, seed, what, packed=True, block=480, hand_over=None, split=True):
    rng = np.random.default_rng(seed)
    starts = [s.start for s in srcs]
    hooks = None
    if hand_over is not None:
        def swap(sess, _):
            t = session(srcs, mix_ch, mix_rate, block=block)
            t.set_state(sess.get_state())
            sess.close()
            return t
        hooks = {hand_over: swap}
    sess = session(srcs, mix_ch, mix_rate, block=block)
    got, sess = drive(sess, srcs, rng, [max(1, s.rate // 150) for s in srcs], block, packed=packed, hooks=hooks, split=split)
    sess.close()
    return check(got, srcs, mix_ch, mix_rate, starts, what), got


# ---------------------------------------------------------------------------------------------------------------------
def s_layout_matrix():
    """Mixers of 1, 2, 3, 4, 6, 8 and 12 channels; sources of 1, 2, 3, 5, 6, 8 and 12 channels in each (more channels than the
    mixer included; a mono mixer takes mono sources only); up-sampling, same-rate and down-sampling rate pairs; random push /
    render splits."""
    rates = [44100, 48000, 22050, 96000, 44100, 48000, 44100]
    for m, mix_ch in enumerate((1, 2, 3, 4, 6, 8, 12)):
        srcs = [Src(ci, rates[(k + m) % len(rates)], start=(37 * k) % 200 if k % 3 else 0, frames=700 + 31 * k, seed=100 * m + k)
                for k, ci in enumerate((1,) * 7 if mix_ch == 1 else (1, 2, 3, 5, 6, 8, 12))]
        run_case(srcs, mix_ch, 48000, 7 + m, f"{mix_ch}-channel mixer", packed=bool(m % 2), block=333)


def s_mixed_layouts_hand_over():
    """Mono, stereo, 5.1 and 12-channel sources in one 8-channel mixer, 40 of them (two warps in some classes), packed 10 ms
    pushes, the state handed to a fresh session in mid-stream."""
    cis = [1, 2, 6, 12] * 10
    rates = [44100, 22050, 48000, 96000, 44100] * 8
    srcs = [Src(ci, r, start=0 if k % 4 else 13 * k, frames=1500 + 7 * k, seed=500 + k) for k, (ci, r) in enumerate(zip(cis, rates))]
    run_case(srcs, 8, 48000, 11, "mixed layouts, 8-channel mixer, hand-over", hand_over=3, split=False)


def s_chain_variants():
    """Filter behind the conversion, filter in front of it with gains on both sides, a gain in front, speed -- in a 6-channel
    mixer with 5.1, stereo, 3-channel and mono sources."""
    srcs = []
    for k, kind in enumerate(("behind", "front", "pre", "speed") * 4):
        ci = (6, 2, 3, 1)[k % 4]
        srcs.append(Src(ci, (44100, 22050, 48000, 96000)[(k // 4) % 4], kind=kind, pre=(0.9, 0.004, -0.6, 1.2)[k % 4],
                        start=0 if k % 2 else 29 * k, frames=800 + 19 * k, seed=700 + k))
    run_case(srcs, 6, 48000, 21, "chain variants, 6-channel mixer", hand_over=2)
    # no filter at all: the lane kernel's filter-free instantiations
    srcs = [Src(ci, 44100, lp=None, gain=g, frames=600 + k, seed=800 + k) for k, (ci, g) in enumerate([(6, 0.5), (5, None), (2, 1.5), (1, None)])]
    run_case(srcs, 6, 48000, 22, "no filter, 6-channel mixer")


def s_split_invariance():
    """1- to 7-frame pushes, single and packed, random renders: the bytes of a one-block render."""
    srcs = [Src(ci, r, frames=400 + 9 * k, seed=900 + k) for k, (ci, r) in enumerate([(6, 44100), (3, 48000), (1, 22050), (8, 96000), (2, 44100)])]
    whole_sess = session(srcs, 6, 48000, block=8192)
    for i, s in enumerate(srcs):
        whole_sess.push(i, s.pcm, end_of_stream=True)
    whole, done = [], False
    while not done:                   # a block ends where a source ends
        block, done = whole_sess.render(8192)
        whole.append(block)
    whole = np.concatenate(whole)
    whole_sess.close()
    check(whole, srcs, 6, 48000, [0] * len(srcs), "one-block render")
    rng = np.random.default_rng(5)
    for packed in (True, False):
        sess = session(srcs, 6, 48000, block=512)
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
    """Held / start, follow, skip, set_amplify and set_volume on multi-slot sources in an 8-channel mixer, with a hand-over."""
    mix_ch, mix_rate = 8, 48000
    srcs = [Src(6, 44100, kind="pre", pre=1.0, frames=6000, seed=1000), Src(5, 32000, kind="pre", pre=1.0, frames=1500, seed=1001),
            Src(8, 48000, kind="pre", pre=1.0, frames=2500, seed=1002), Src(3, 22050, kind="pre", pre=1.0, frames=1200, seed=1003),
            Src(12, 44100, kind="pre", pre=1.0, frames=6000, seed=1004)]
    starts = [0, HELD, HELD, 0, 0]
    sess = session(srcs, mix_ch, mix_rate, starts=starts, block=256)
    sess.follow(1, 0)                 # 1 plays behind 0; 2 is added by hand
    sess.set_volume(3, 0.5)           # before anything was pulled: every frame of source 3 carries 0.5
    sess.set_amplify(4, 0.25)         # the gain behind the conversion of source 4, from the first block on
    got, marks, pos = [], {}, [0] * 5      # source 0 is skipped in round 7, long before its input would end
    for rnd in range(400):
        if rnd == 3:
            marks["T2"] = sum(b.size for b in got) // mix_ch
            sess.start(2)
        if rnd == 5:
            t = session(srcs, mix_ch, mix_rate, starts=starts, block=256)
            t.set_state(sess.get_state())
            sess.close()
            sess = t
        if rnd == 7:
            marks["T0"] = sum(b.size for b in got) // mix_ch
            sess.skip(0)
        blocks, eos = [], []
        for i, s in enumerate(srcs):
            total = s.pcm.size // s.ci
            k = 0 if (i == 0 and rnd >= 7) else min(s.rate // 100, total - pos[i])
            blocks.append(s.pcm[s.ci * pos[i]: s.ci * (pos[i] + k)])
            pos[i] += k
            eos.append(pos[i] == total and not (i == 0 and rnd >= 7))
        sess.push_packed(blocks, eos)
        ended = False
        while True:
            block, ended = sess.render(256)
            got.append(block)
            if block.size == 0 or ended:
                break
        if ended:
            break
    sess.close()
    got = np.concatenate(got)
    n0 = marks["T0"]                                              # outputs of source 0 rendered before the skip (it started at 0)
    fpos = min(((n0 - 1) * 147) // 160 + 2, pos[0])               # what its converter had pulled: its whole input now
    pcms = [s.pcm for s in srcs]
    pcms[0] = pcms[0][:srcs[0].ci * fpos]
    real = [s.chain(mix_ch, mix_rate, p, pre=(0.5 if i == 3 else None)) for i, (s, p) in enumerate(zip(srcs, pcms))]
    real[4] = rb.UniformSourceIterator(rb.TestSource(pcms[4], 12, 44100).amplify(1.0), mix_ch, mix_rate).low_pass(srcs[4].lp).amplify(0.25)
    per = [oracle.chain_uniform(to_oracle(x), mix_ch, mix_rate) for x in real]
    len0 = per[0].size // mix_ch
    joined = [0, len0, marks["T2"], 0, 0]
    want = slot_expected(per, joined, srcs, mix_ch, mix_rate)
    assert_bit_exact(got, want[:got.size], "held / follow / skip / volume / amplify on multi-slot sources")
    assert got.size == want.size or not np.any(want[got.size:]), "tail"
    assert_close_peak(got, oracle.mixer([to_oracle(x, st * mix_ch) for x, st in zip(real, joined)], mix_ch, mix_rate)[:got.size], 1e-5, "sequential mixer")


def s_volume_changes():
    """set_volume in mid-stream on a 5.1 source and on a 3-channel one with the filter in front: every frame keeps the factor it
    was pulled with by the converter, on every slot row of the source."""
    mix_ch, mix_rate = 6, 48000
    srcs = [Src(6, 44100, kind="pre", pre=1.0, frames=5000, seed=1100), Src(3, 22050, kind="front", pre=0.8, mid=1.0, frames=2500, seed=1101)]
    vols = {2: 0.5, 4: 0.25, 6: 1.5}
    total = [int(rb.plan(s.chain(mix_ch, mix_rate, s.pcm), mix_ch, mix_rate)[0]) for s in srcs]
    gains = [np.ones(s.pcm.size // s.ci, np.float32) for s in srcs]
    pulled, pushed, done, vol = [0, 0], [0, 0], [0, 0], [1.0, 1.0]
    got = []
    with session(srcs, mix_ch, mix_rate, block=240) as sess:
        ended, rnd = False, 0
        while not ended:
            if rnd in vols:
                for i in range(2):
                    vol[i] = vols[rnd]
                    sess.set_volume(i, vol[i])
            blocks, eos = [], []
            for i, s in enumerate(srcs):
                L = s.pcm.size // s.ci
                k = min(s.rate // 100, L - pushed[i])
                blocks.append(s.pcm[s.ci * pushed[i]: s.ci * (pushed[i] + k)])
                pushed[i] += k
                eos.append(pushed[i] == L)
            sess.push_packed(blocks, eos)
            while True:
                block, ended = sess.render(240)
                got.append(block)
                if block.size == 0:
                    break
                for i, s in enumerate(srcs):
                    o = min(done[i] + block.size // mix_ch, total[i])
                    if o > done[i]:
                        g = math.gcd(s.rate, mix_rate)
                        p_new = min(((o - 1) * (s.rate // g)) // (mix_rate // g) + 2, pushed[i])
                        gains[i][pulled[i]:p_new] = np.float32(vol[i])
                        pulled[i], done[i] = p_new, o
                if ended:
                    break
            rnd += 1
            assert rnd < 1000
    got = np.concatenate(got)
    s0, s1 = srcs
    x0 = (s0.pcm.reshape(-1, 6) * gains[0][:, None]).reshape(-1)
    y0 = oracle.chain_uniform(to_oracle(rb.UniformSourceIterator(rb.TestSource(x0, 6, 44100), mix_ch, mix_rate).low_pass(s0.lp).amplify(s0.gain)), mix_ch, mix_rate)
    f1 = oracle.chain_uniform(to_oracle(rb.TestSource(s1.pcm, 3, 22050).amplify(0.8).low_pass(s1.lp)), 3, 22050)
    x1 = (f1.reshape(-1, 3) * gains[1][:, None]).reshape(-1)
    y1 = oracle.chain_uniform(to_oracle(rb.UniformSourceIterator(rb.TestSource(x1, 3, 22050), mix_ch, mix_rate).amplify(s1.gain)), mix_ch, mix_rate)
    want = slot_expected([y0, y1], [0, 0], srcs, mix_ch, mix_rate)
    assert all(np.unique(g).size > 2 for g in gains)
    assert_bit_exact(got, want[:got.size], "volume changes on every slot row")


def s_today_shapes_blob():
    """Mono and stereo mixers keep the version-5 blob: 32 + 112 bytes per source plus the FIFO contents, one record per source."""
    for mix_ch, cis in ((2, [1, 2, 1]), (1, [1, 1])):
        srcs = [Src(ci, 44100, frames=500, seed=1200 + k) for k, ci in enumerate(cis)]
        with session(srcs, mix_ch, 48000) as s:
            blob = s.get_state()
            assert int.from_bytes(blob[4:8], "little") == 5 and len(blob) == 32 + 112 * len(cis)
            s.push_packed([x.pcm[:x.ci * 100] for x in srcs])
            blob = s.get_state()
            assert len(blob) == 32 + 112 * len(cis) + 4 * sum(100 * ci for ci in cis)
    # other layouts: one record per slot row and version 6; a blob from another layout is refused
    srcs = [Src(6, 44100, frames=500, seed=1300), Src(2, 44100, frames=500, seed=1301)]
    with session(srcs, 6, 48000) as a, session([Src(2, 44100), Src(6, 44100)], 6, 48000) as b, session(srcs[::-1][:1] + srcs[1:], 6, 48000) as c:
        blob = a.get_state()
        assert int.from_bytes(blob[4:8], "little") == 6 and int.from_bytes(blob[8:12], "little") == 4   # 3 + 1 rows
        for other in (b, c):
            try:
                other.set_state(blob)
            except capi.RodioB200Error as e:
                assert e.status == capi.RB_ERR_INVALID_ARGUMENT
            else:
                raise AssertionError("a blob of another layout was accepted")


def s_coverage():
    """Every slot class of a layout runs fast tiles (the CPU build's per-class counters): no case passes on slow tiles alone."""
    import ctypes as C
    srcs = [Src(ci, r, frames=3000, seed=1400 + k) for k, (ci, r) in enumerate([(6, 44100), (5, 48000), (1, 22050), (12, 96000), (2, 44100), (3, 32000)])]
    sess = session(srcs, 8, 48000)
    got, sess = drive(sess, srcs, np.random.default_rng(31), [s.rate // 100 for s in srcs], 480, split=False)
    out = (C.c_uint64 * 64)()
    n = capi.lib().rb_session_emu_fast_tiles(sess._h, out, 64)
    sess.close()
    check(got, srcs, 8, 48000, [0] * len(srcs), "coverage layout")
    n_classes = len(slot_classes(srcs, 8, 48000))
    assert n == n_classes, (n, n_classes)
    assert all(out[k] > 10 for k in range(n)), list(out[:n])


def s_refusals():
    """13 channels; more than one channel in a mono mixer; a source whose conversion pads channels behind a non-finite gain or
    filter (rodio puts NaN there)."""
    U = capi.RB_ERR_UNSUPPORTED

    def refused(make, status=U):
        try:
            make().close()
        except capi.RodioB200Error as e:
            assert e.status == status, e
        else:
            raise AssertionError("accepted")
    z = np.zeros(0, np.float32)
    refused(lambda: rb.Session([rb.UniformSourceIterator(rb.TestSource(z, 13, 44100), 2, 48000)], 48000, mixer_channels=2))
    refused(lambda: rb.Session([rb.UniformSourceIterator(rb.TestSource(z, 2, 44100), 13, 48000)], 48000, mixer_channels=13))
    for ci in (2, 6):
        refused(lambda: rb.Session([rb.UniformSourceIterator(rb.TestSource(z, ci, 44100), 1, 48000)], 48000, mixer_channels=1))
    inf = float("inf")
    for ci, mix_ch in ((1, 3), (2, 6), (5, 8)):           # padded: amplify(inf), amplify(nan), a filter with a NaN coefficient
        refused(lambda: rb.Session([rb.UniformSourceIterator(rb.TestSource(z, ci, 44100), mix_ch, 48000).low_pass(300).amplify(inf)], 48000, mixer_channels=mix_ch))
        refused(lambda: rb.Session([rb.UniformSourceIterator(rb.TestSource(z, ci, 44100), mix_ch, 48000).amplify(float("nan"))], 48000, mixer_channels=mix_ch))
        refused(lambda: rb.Session([rb.UniformSourceIterator(rb.TestSource(z, ci, 44100), mix_ch, 48000).low_pass_with_q(300, 1e-45)], 48000, mixer_channels=mix_ch))
    # not padded: the same gain is served (every output channel carries a source channel)
    for ci, mix_ch in ((2, 2), (1, 2), (6, 2), (1, 1)):
        rb.Session([rb.UniformSourceIterator(rb.TestSource(z, ci, 44100), mix_ch, 48000).amplify(inf)], 48000, mixer_channels=mix_ch).close()
    # a padded source cannot get a non-finite gain later either
    with rb.Session([rb.UniformSourceIterator(rb.TestSource(z, 2, 44100), 6, 48000).amplify(1.0)], 48000, mixer_channels=6) as s:
        try:
            s.set_amplify(0, inf)
        except capi.RodioB200Error as e:
            assert e.status == U
        else:
            raise AssertionError("set_amplify(inf) on a padded source was accepted")
        s.set_amplify(0, 2.0)


def s_fifo_errors():
    """A multi-slot source's FIFO refuses a push it cannot hold and a push after its end of stream."""
    mk = lambda ci, r, mc: rb.UniformSourceIterator(rb.TestSource(np.zeros(0, np.float32), ci, r), mc, 48000).low_pass(200)
    with rb.Session([mk(6, 44100, 6)], 48000, fifo_frames=64, max_block_frames=64, mixer_channels=6) as s:
        s.push(0, noise(6 * 64, 1))
        try:
            s.push(0, noise(6, 2))
        except rb.RodioB200Error as e:
            assert "FIFO" in str(e) or "full" in str(e).lower(), str(e)
        else:
            raise AssertionError("a push beyond the FIFO was accepted")
        out, ended = s.render(64)
        assert out.size > 0 and not ended
        s.push(0, noise(60, 3), end_of_stream=True)
        try:
            s.push(0, noise(6, 4))
        except rb.RodioB200Error:
            pass
        else:
            raise AssertionError("a push after end_of_stream was accepted")


SCENARIOS = {"layout_matrix": s_layout_matrix, "mixed_layouts_hand_over": s_mixed_layouts_hand_over, "chain_variants": s_chain_variants,
             "split_invariance": s_split_invariance, "controls": s_controls, "volume_changes": s_volume_changes,
             "today_shapes_blob": s_today_shapes_blob, "coverage": s_coverage, "refusals": s_refusals, "fifo_errors": s_fifo_errors}

if __name__ == "__main__":
    for name in (sys.argv[1:] or list(SCENARIOS)):
        SCENARIOS[name]()
        print("ok", name, flush=True)
