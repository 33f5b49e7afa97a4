"""Adapters on the MixerSource itself: Amplify(Limit(Amplify(MixerSource))) -- rb_batch_set_master / rb_session_set_master,
served by k_master (rodio_b200/csrc/rb_master.cu) in place on the rendered mix.

The reference is rodio's pull model: the oracle's mixer, whose positions where MixerSource::next() returns None (gaps: no source
playing, a later Mixer::add still scheduled) are not pulled through the chain; the oracle's Amplify / Limit run over the
active samples as one sequence, a SamplesBuffer of the mixer's format.  Sessions run on the CPU through the library's host code
over the mock CUDA runtime (tests/emu), in a subprocess: `python tests/test_master_chain.py <scenario>`."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(HERE, "emu")

if __name__ == "__main__":      # emulator scenario: the library path is swapped in this process only
    sys.path[:0] = [ROOT, HERE, EMU]
    import build_emu
    import rodio_b200._capi as capi
    capi.LIB_PATH = build_emu.HOST_LIB

import oracle                                                      # noqa: E402
import rodio_b200 as rb                                            # noqa: E402
from rodio_b200 import capi                                        # noqa: E402
from rodio_b200.source import LimitSettings, amplify_effect, limit_effect   # noqa: E402
from helpers import assert_bit_exact, assert_close_peak, noise, to_oracle   # noqa: E402

PRESETS = {"default": LimitSettings.default(), "dynamic_content": LimitSettings.dynamic_content(),
           "broadcast": LimitSettings.broadcast(), "mastering": LimitSettings.mastering(),
           "live_performance": LimitSettings.live_performance(), "gaming": LimitSettings.gaming()}


def master_fx(settings=None, pre=None, post=None, limit=True):
    fx = [] if pre is None else [amplify_effect(pre)]
    if limit:
        fx.append(limit_effect(settings))
    return fx + ([] if post is None else [amplify_effect(post)])


def active_mask(streams, ch, rate, mix_len):
    """Positions where MixerSource::next() is Some: some source plays (joins on the next frame boundary, mixer.rs:175-183)."""
    act = np.zeros(mix_len + 1, np.int64)
    for s in streams:
        n = oracle.chain_uniform(s, ch, rate).size
        if n:
            st = -(-s.mix_start // ch) * ch
            act[st] += 1
            act[min(st + n, mix_len)] -= 1
    return np.cumsum(act)[:-1] > 0


def mastered(mix, active, ch, rate, fx):
    """The chain over the active samples as one sequence; gap positions stay 0.0."""
    out = np.zeros_like(mix)
    seq = np.ascontiguousarray(mix[active])
    if seq.size:
        y, _, _ = oracle.chain(oracle.Stream(pcm=seq, channels=ch, sample_rate=rate, effects=list(fx), span_len=seq.size))
        assert y.size == seq.size
        out[active] = y
    return out


def oracle_master(streams, ch, rate, fx):
    mix, gaps = oracle.mixer(streams, ch, rate, return_gaps=True)
    act = active_mask(streams, ch, rate, mix.size)
    assert int((~act).sum()) == gaps
    return mastered(mix, act, ch, rate, fx), act


def gap_streams(ch, rate, n_gaps, seed=0):
    """Sources of the mixer's format (and one at 44.1 kHz) with late joins that leave `n_gaps` gaps."""
    srcs, starts = [], []
    t = 0
    for g in range(n_gaps + 1):
        frames = 700 + 37 * g
        for k in range(2):
            x = noise(frames * ch, seed + 10 * g + k, 0.9)
            srcs.append(rb.TestSource(x, ch, rate if k == 0 else 44100))
            starts.append((t + 5 * k) * ch)
        t += frames + 120 + 13 * g        # the next join leaves a gap behind the longest source of this group
    return [rb.UniformSourceIterator(s, ch, rate) for s in srcs], starts


# ---------------------------------------------------------------- CPU: the reference
@pytest.mark.parametrize("ch", [1, 2, 4])
@pytest.mark.parametrize("n_gaps", [0, 1, 2])
def test_reference_gaps_and_sequence(ch, n_gaps):
    """The oracle mixer's gaps are exactly the positions no source covers; the mastered reference leaves them at 0.0, and
    without gaps it is the chain over the whole mix."""
    srcs, starts = gap_streams(ch, 48000, n_gaps, seed=100 * ch)
    streams = [to_oracle(s, st) for s, st in zip(srcs, starts)]
    mix = oracle.mixer(streams, ch, 48000)
    for name, st in PRESETS.items():
        for pre, post in ((None, None), (0.8, 1.5)):
            fx = master_fx(st, pre, post)
            got, act = oracle_master(streams, ch, 48000, fx)
            assert (~act).sum() >= n_gaps * 40 * ch and np.all(mix[~act] == 0.0)
            assert np.all(got[~act].view(np.uint32) == 0)
            if n_gaps == 0:
                want, _, _ = oracle.chain(oracle.Stream(pcm=mix, channels=ch, sample_rate=48000, effects=fx, span_len=mix.size))
                assert_bit_exact(got, want, f"{name} ch={ch}")
            else:   # a gap is not pulled: the run behind it continues the limiter, it does not restart it
                first = np.nonzero(~act)[0][0]
                restart = mastered(mix[first:], act[first:], ch, 48000, fx)
                assert not np.array_equal(got[first:], restart), name


def test_one_source_mixer_limit_equals_source_limit():
    """mixer(ch, rate) with one source of its format, .limit() on the MixerSource == .limit() on the source, by value (the
    mixer's sum from +0.0 turns -0.0 into +0.0)."""
    for ch in (1, 2):
        x = noise(ch * 9000, 7 + ch, 1.0)
        x[: 2 * ch] = -0.0
        src = rb.SamplesBuffer(ch, 48000, x)
        for st in PRESETS.values():
            want, _, _ = oracle.chain(to_oracle(src.limit(st)))
            got, _ = oracle_master([to_oracle(src)], ch, 48000, master_fx(st))
            assert np.array_equal(got, want) and np.abs(got).max() < np.abs(x).max()


# ---------------------------------------------------------------- CPU: sessions on the emulator
SCENARIOS = ["random_split_mono", "random_split_stereo", "held_follow_and_gap", "state_handover", "errors"]


@pytest.fixture(scope="module")
def hostemu(built):
    sys.path[:0] = [EMU]
    import build_emu
    return build_emu.host_lib()


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_master_on_the_emulator(hostemu, scenario):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), scenario], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and f"ok {scenario}" in r.stdout, (r.stdout + r.stderr)[-3000:]


def _chain(ch_mix, rate, lp=None, gain=None, ch_in=None):
    s = rb.UniformSourceIterator(rb.TestSource(np.zeros(0, np.float32), ch_in or ch_mix, rate), ch_mix, 48000)
    if lp:
        s = s.low_pass(lp)
    return s.amplify(gain) if gain is not None else s


def _with_pcm(chain_src, pcm):
    """The same chain over real PCM (for the oracle)."""
    s = rb.TestSource(pcm, chain_src.base_channels, chain_src.base_rate)
    for e in chain_src.effects:
        s = s._with(e)
    return s


def _drive(sess, pcms, ch_in, rng, max_block, hooks=None):
    """Random pushes and renders of 1..max_block frames until the session has ended."""
    pos, got, rnd = [0] * len(pcms), [], 0
    while True:
        if hooks and rnd in hooks:
            sess = hooks[rnd](sess) or sess
        blocks, eos = [], []
        for i, (p, ci) in enumerate(zip(pcms, ch_in)):
            k = min(int(rng.integers(0, 600)), p.size // ci - pos[i])
            blocks.append(p[ci * pos[i]: ci * (pos[i] + k)])
            pos[i] += k
            eos.append(pos[i] == p.size // ci)
        sess.push_packed(blocks, eos)
        while True:
            block, ended = sess.render(int(rng.integers(1, max_block + 1)))
            got.append(block)
            if block.size == 0 or ended:
                break
        if ended:
            return np.concatenate(got), sess
        rnd += 1
        assert rnd < 100000


def _unsplit(make, pcms):
    with make() as s:
        s.push_packed(pcms, [True] * len(pcms))
        out = []
        while True:
            b, e = s.render()
            out.append(b)
            if e or b.size == 0:
                return np.concatenate(out)


def _random_split(ch):
    rates = [44100, 48000, 22050, 44100, 48000] * 3
    ch_in = [1 if (i % 3 == 0) else ch for i in range(len(rates))]
    chains = [_chain(ch, r, lp=900 if i % 2 else None, gain=0.9, ch_in=ci) for i, (r, ci) in enumerate(zip(rates, ch_in))]
    pcms = [noise(ci * (3000 + 211 * i), 500 + i, 0.7) for i, ci in enumerate(ch_in)]
    fx = master_fx(LimitSettings.mastering(), pre=1.7, post=0.9)
    make = lambda: rb.Session(chains, 48000, fifo_frames=8192, max_block_frames=700, mixer_channels=ch, master=fx)
    whole = _unsplit(make, pcms)
    streams = [to_oracle(_with_pcm(c, p)) for c, p in zip(chains, pcms)]
    want, _ = oracle_master(streams, ch, 48000, fx)
    assert_close_peak(whole, want, 1e-5, f"session ch={ch} vs oracle")
    assert np.abs(whole).max() < np.abs(oracle.mixer(streams, ch, 48000)).max()    # the limiter acted
    for seed in range(3):
        with make() as s:
            got, _ = _drive(s, pcms, ch_in, np.random.default_rng(seed), 700)
        assert_bit_exact(got, whole, f"ch={ch} split seed {seed}")


def s_random_split_mono():
    _random_split(1)


def s_random_split_stereo():
    _random_split(2)


def s_held_follow_and_gap():
    """A plays; D is declared to join at frame 20000, after A has ended: a gap the chain is not pulled through.  B is held and
    started once D has ended and nothing plays (the timeline stands still meanwhile); C follows B."""
    fx = master_fx(LimitSettings.broadcast(), post=1.25)
    chains = [_chain(1, 44100, gain=1.1), _chain(1, 48000), _chain(1, 22050, lp=700), _chain(1, 48000, gain=0.8)]
    pcms = [noise(4000, 1, 0.9), noise(3000, 2, 0.9), noise(1500, 3, 0.9), noise(2000, 4, 0.9)]
    with rb.Session(chains, 48000, fifo_frames=8192, max_block_frames=512, mix_starts=[0, capi.RB_SESSION_HELD, capi.RB_SESSION_HELD, 20000],
                    master=fx) as s:
        s.follow(2, 1)
        out = []
        s.push(0, pcms[0], end_of_stream=True)
        s.push(3, pcms[3], end_of_stream=True)
        while True:
            b, e = s.render(300)
            if b.size == 0:
                break
            out.append(b)
        t1 = sum(b.size for b in out)
        for _ in range(3):      # nothing plays: the timeline stands still
            b, e = s.render(300)
            assert b.size == 0 and not e
        s.start(1)
        s.push(1, pcms[1], end_of_stream=True)
        s.push(2, pcms[2], end_of_stream=True)
        while True:
            b, e = s.render(300)
            out.append(b)
            if e:
                break
        got = np.concatenate(out)
    assert t1 == 22000
    b_len = oracle.chain_uniform(to_oracle(_with_pcm(chains[1], pcms[1])), 1, 48000).size
    starts = [0, t1, t1 + b_len, 20000]
    streams = [to_oracle(_with_pcm(c, p), st) for c, p, st in zip(chains, pcms, starts)]
    want, act = oracle_master(streams, 1, 48000, fx)
    assert (~act).sum() > 0, "the scenario must leave a gap"
    assert got.size == want.size
    assert np.all(got[~act].view(np.uint32) == 0)
    assert_close_peak(got, want, 1e-5, "held / follow / gap")


def s_state_handover():
    """get_state / set_state mid-stream into a fresh session with the same master chain; blob sizes and refusals."""
    ch = 2
    chains = [_chain(ch, r, lp=800, gain=0.8, ch_in=ci) for r, ci in ((44100, 1), (48000, 2), (22050, 2), (44100, 2))]
    pcms = [noise(ci * 6000, 40 + i, 0.9) for i, ci in enumerate((1, 2, 2, 2))]
    fx = master_fx(LimitSettings.gaming(), pre=1.4)
    mk = lambda m: rb.Session(chains, 48000, fifo_frames=8192, max_block_frames=600, mixer_channels=ch, master=m)
    whole = _unsplit(lambda: mk(fx), pcms)
    sa, sb, plain, other = mk(fx), mk(fx), mk(()), mk(master_fx(LimitSettings.gaming(), pre=1.5))

    def hand_over(s):
        blob = s.get_state()
        assert int.from_bytes(blob[20:24], "little") == 1
        for dst, src_blob in ((plain, blob), (other, blob), (sb, plain.get_state())):
            try:
                dst.set_state(src_blob)
                raise AssertionError("a blob crossed to a session with another master chain")
            except capi.RodioB200Error as e:
                assert e.status == capi.RB_ERR_INVALID_ARGUMENT
        sb.set_state(blob)
        return sb
    got, _ = _drive(sa, pcms, [1, 2, 2, 2], np.random.default_rng(9), 600, hooks={3: hand_over})
    for s in (sa, sb, plain, other):
        s.close()
    assert_bit_exact(got, whole, "state hand-over")
    # a session without a master chain: the blob has no master record and its header flag stays 0
    ns = len(chains)
    with mk(()) as p:
        blob = p.get_state()
        assert int.from_bytes(blob[20:24], "little") == 0
        assert len(blob) == 32 + ns * 112      # header + one record per source, FIFOs empty: the layout of before
    with mk(fx) as p:
        assert len(p.get_state()) == 32 + ns * 112 + 140   # + chain parameters, channels, integ[12], peak[12]


def s_errors():
    U, S, I = capi.RB_ERR_UNSUPPORTED, capi.RB_ERR_STATE, capi.RB_ERR_INVALID_ARGUMENT
    A, L = amplify_effect(0.5), limit_effect()
    bad = [[A, A, A], [L, L], [L, A, A], [A, A, L], [L, A, L],
           [rb.source.Effect.make(capi.RB_FX_AGC, f32=[1.0, 7.0])], [A, rb.source.Effect.make(capi.RB_FX_LOW_PASS, u32=[500], f32=[0.5])]]
    chains = [_chain(1, 44100, gain=1.0)]
    for fx in bad:
        with rb.Session(chains, 48000) as s:
            try:
                s.set_master(fx)
                raise AssertionError(f"accepted {[e.kind for e in fx]}")
            except capi.RodioB200Error as e:
                assert e.status == U, e
    for fx in ([A], [L], [A, L], [L, A], [A, L, A], [A, A], []):
        with rb.Session(chains, 48000) as s:
            s.set_master(fx)
    with rb.Session(chains, 48000, master=[L]) as s:
        s.push(0, noise(2000, 1), end_of_stream=True)
        s.set_master([A])          # nothing rendered yet
        s.render(100)
        for fx in ([L], []):
            try:
                s.set_master(fx)
                raise AssertionError("set_master after a render")
            except capi.RodioB200Error as e:
                assert e.status == S
    L_ = capi.lib()
    assert L_.rb_batch_set_master(None, None, 0) == I and L_.rb_session_set_master(None, None, 0) == I
    with rb.Session(chains, 48000) as s:
        assert L_.rb_session_set_master(s._h, None, 1) == I
    # batches the host code can plan without a device: the lane kernel's shape
    srcs = [rb.UniformSourceIterator(rb.TestSource(noise(4000, 3 + i), 1, 44100), 1, 48000).amplify(0.5) for i in range(40)]
    with rb.Batch(srcs, 1, 48000, flags=capi.RB_FUSED_LANES) as b:
        base = b.launches_per_render
        for fx in bad:
            assert L_.rb_batch_set_master(b._h, rb.source.effect_records(fx), len(fx)) == U
        assert L_.rb_batch_set_master(b._h, rb.source.effect_records([A, L, A]), 3) == 0
        assert b.launches_per_render == base + 1 and b.kernel_family == 2
        assert L_.rb_batch_set_master(b._h, None, 0) == 0 and b.launches_per_render == base


# ---------------------------------------------------------------- GPU
def _limit_tile_reference(ctx, mix, act, ch, rate, settings, pre, post):
    """The existing limiter (k_limit_tile, one kernel per adapter): SamplesBuffer(active samples).amplify(a).limit(s).amplify(b)."""
    seq = np.ascontiguousarray(mix[act])
    s = rb.SamplesBuffer(ch, rate, seq)
    if pre is not None:
        s = s.amplify(pre)
    s = s.limit(settings)
    if post is not None:
        s = s.amplify(post)
    with rb.Batch([s], ch, rate, flags=capi.RB_NO_FUSION, ctx=ctx) as b:
        b.upload_all()
        return b.render_mix()


def _check_batch(ctx, srcs, starts, ch, fx_args, flags=0, family=None, oracle_check=True):
    settings, pre, post = fx_args
    fx = master_fx(settings, pre, post)
    with rb.Batch(srcs, ch, 48000, flags=flags, mix_starts=starts, ctx=ctx) as b:
        fam, grp, base = b.kernel_family, b.mix_group, b.launches_per_render
        b.upload_all()
        raw = b.render_mix()
    with rb.Batch(srcs, ch, 48000, flags=flags, mix_starts=starts, ctx=ctx, master=fx) as b:
        assert (b.kernel_family, b.mix_group, b.launches_per_render) == (fam, grp, base + 1)
        if family is not None:
            assert fam == family, fam
        b.upload_all()
        got = b.render_mix()
        again = b.render_mix()
        assert_bit_exact(again, got, "second render")
        assert_bit_exact(b.read_mix(0, got.size), got, "read_mix")
    streams = [to_oracle(s, st) for s, st in zip(srcs, starts or [0] * len(srcs))]
    act = active_mask(streams, ch, 48000, raw.size)
    assert np.all(got[~act].view(np.uint32) == 0)
    want = _limit_tile_reference(ctx, raw, act, ch, 48000, settings, pre, post)
    assert np.array_equal(got[act], want), "k_master != k_limit_tile"
    if oracle_check:
        ref, _ = oracle_master(streams, ch, 48000, fx)
        assert_close_peak(got, ref, 1e-5, "vs oracle")
    return got, raw


@pytest.mark.gpu
@pytest.mark.parametrize("ch", [1, 2, 4, 12])
@pytest.mark.parametrize("n_gaps", [0, 2])
def test_master_equals_limit_tile(ctx, ch, n_gaps):
    srcs, starts = gap_streams(ch, 48000, n_gaps, seed=7 * ch)
    for i, st in enumerate(PRESETS.values()):
        for pre, post in ((None, None), (1.9, 0.7)):
            _check_batch(ctx, srcs, starts, ch, (st, pre, post), flags=capi.RB_NO_FUSION if i % 2 else 0)


def _cfg3(n, frames, ch=1, lp=200, gain=1.2, seed=31000):
    srcs = []
    for s in range(n):
        src = rb.UniformSourceIterator(rb.TestSource(noise(frames * ch, seed + s), ch, 44100), ch, 48000)
        if lp:
            src = src.low_pass(lp)
        srcs.append(src.amplify(gain))
    return srcs


@pytest.mark.gpu
def test_master_behind_k_fused_hot_cfg3(ctx):
    """The cfg3 batch (4096 x 2 s of 44.1 kHz mono, low_pass(200), amplify(1.2)) with .limit(mastering)."""
    srcs = _cfg3(4096, 88200)
    got, raw = _check_batch(ctx, srcs, None, 1, (LimitSettings.mastering(), None, None), family=1, oracle_check=False)
    nz = raw != 0
    assert np.any(np.abs(got[nz]) < np.abs(raw[nz]) * 0.999), "the limiter never reduced the gain"


@pytest.mark.gpu
@pytest.mark.parametrize("flags,family,gaps", [(capi.RB_FUSED_LANES, 2, True), (capi.RB_FUSED_DUO, 3, False),
                                               (capi.RB_MIX_EXACT_ORDER, None, False), (capi.RB_NO_FUSION, -1, True), (0, None, True)])
def test_master_behind_every_family(ctx, flags, family, gaps):
    srcs = _cfg3(256, 4410, seed=900)
    starts = [0 if i < 200 else 6000 for i in range(256)] if gaps else None
    _check_batch(ctx, srcs, starts, 1, (LimitSettings.live_performance(), 2.0, 0.8), flags=flags, family=family)


@pytest.mark.gpu
def test_master_behind_effect_chain_cfg4(ctx):
    sys.path[:0] = [HERE]
    from test_bench_geometries_gpu import cfg4_sources
    _check_batch(ctx, cfg4_sources(64, 4800), None, 2, (LimitSettings.dynamic_content(), None, 1.1), family=5, oracle_check=False)


@pytest.mark.gpu
def test_amplify_only_exact_order_is_bit_exact(ctx):
    srcs = _cfg3(64, 4410, seed=77)
    starts = [0 if i < 40 else 9000 for i in range(64)]
    fx = [amplify_effect(0.37), amplify_effect(1.3)]
    with rb.Batch(srcs, 1, 48000, flags=capi.RB_MIX_EXACT_ORDER, mix_starts=starts, ctx=ctx, master=fx) as b:
        b.upload_all()
        got = b.render_mix()
    streams = [to_oracle(s, st) for s, st in zip(srcs, starts)]
    mix = oracle.mixer(streams, 1, 48000)
    want = mastered(mix, active_mask(streams, 1, 48000, mix.size), 1, 48000, fx)
    assert_bit_exact(got, want, "amplify-only master, exact order")


@pytest.mark.gpu
@pytest.mark.parametrize("ch", [1, 2])
def test_session_on_device_equals_lanes_batch(ctx, ch):
    rates = [44100, 22050] * 20
    chains = [_chain(ch, r, lp=700, gain=0.9) for r in rates]
    pcms = [noise(ch * (20000 + 331 * i), 70 + i, 0.8) for i in range(len(rates))]
    fx = master_fx(LimitSettings.mastering(), pre=2.0)
    srcs = [_with_pcm(c, p) for c, p in zip(chains, pcms)]
    with rb.Batch(srcs, ch, 48000, flags=capi.RB_FUSED_LANES, ctx=ctx, master=fx) as b:
        assert b.kernel_family == 2
        b.upload_all()
        want = b.render_mix()
    mk = lambda: rb.Session(chains, 48000, fifo_frames=32768, max_block_frames=1000, mixer_channels=ch, master=fx, ctx=ctx)
    sb = mk()

    def hand_over(s):
        sb.set_state(s.get_state())
        return sb
    with mk() as sa:
        got, _ = _drive(sa, pcms, [ch] * len(pcms), np.random.default_rng(ch), 1000, hooks={5: hand_over})
    sb.close()
    assert_bit_exact(got, want, "device session vs RB_FUSED_LANES batch")


@pytest.mark.gpu
def test_allreduce_refuses_a_master_chain(ctx):
    import ctypes as C
    srcs = _cfg3(8, 4410)
    h = C.c_void_p()
    ctxs = (C.c_void_p * 1)(ctx._h)
    if capi.lib().rb_comm_init_all(ctxs, 1, C.byref(h)) != 0:
        pytest.skip("no one-GPU communicator (NCCL not loadable)")
    try:
        with rb.Batch(srcs, 1, 48000, ctx=ctx, master=master_fx()) as b:
            b.upload_all()
            arr = (C.c_void_p * 1)(b._h)
            assert capi.lib().rb_batch_render_mix_allreduce(arr, 1, h) == capi.RB_ERR_UNSUPPORTED
    finally:
        capi.lib().rb_comm_destroy(h)


if __name__ == "__main__":
    for name in sys.argv[1:]:
        globals()["s_" + name]()
        print("ok", name)
