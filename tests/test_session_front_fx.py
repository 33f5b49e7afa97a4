"""Push programs in streaming sessions -- fade_in / fade_out / linear_gain_ramp / take_duration / distortion applied as sources are
pushed -- and rb_session_push_silence for Player::pause (tests/emu/front_fx_scenarios.py): on the CPU through the host-emulated
library, on the H100 through the real one, bit for bit against the oracle's chains summed in the documented slot order and within
1e-5 * peak of the oracle's sequential mixer."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
sys.path[:0] = [EMU]

SCENARIOS = ["adapters", "mid_frame_takes", "program_variants", "split_invariance", "controls", "pause", "large_pushes", "refusals"]


@pytest.fixture(scope="module")
def hostemu(built):
    import build_emu
    return build_emu.host_lib()


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_front_fx_on_the_emulator(hostemu, scenario):
    r = subprocess.run([sys.executable, os.path.join(EMU, "front_fx_scenarios.py"), scenario], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and f"ok {scenario}" in r.stdout, (r.stdout + r.stderr)[-3000:]


@pytest.fixture(scope="module")
def front_fx(ctx):
    import layout_scenarios as L
    import front_fx_scenarios as F
    L.CTX["ctx"] = ctx
    yield F
    L.CTX["ctx"] = None


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_front_fx_on_the_device(front_fx, scenario):
    front_fx.SCENARIOS[scenario]()


@pytest.mark.gpu
def test_session_front_fx_at_scale(front_fx):
    """1024 stereo sources into a 48 kHz stereo mixer, each fade_in(200 ms).take_duration(...) with the fade-out filter; 10 ms packed
    pushes and renders, one state hand-over, pauses on a tenth of the sources.  The 44.1 kHz sources take 350 ms, one run of the
    mixer's conversion; the paused tenth is at 48 kHz with a 1.5 s take (rodio restarts a resampling conversion behind a paused take,
    which sessions refuse)."""
    F = front_fx
    L = F.L
    srcs, pend = [], {}
    for k in range(1024):
        paused = k % 10 == 0
        rate = 48000 if paused else 44100
        d = F.take_ns(rate, 2, 1500 if paused else 350)
        srcs.append(F.FSrc(2, rate, [("fade_in", 200 * F.MS), ("take", d, True)], kind="pre", pre=1.0, lp=None if k % 3 else 700,
                           frames=(rate * 16) // 10 - 7 * (k % 50), start=0 if k % 7 else 3 * k, seed=30000 + k))
        if paused:
            pend[k] = (4800 + 37 * (k % 11), 2400 + k)       # (frame of the source, frames of silence)
    pauses = dict(pend)
    sess = L.session(srcs, 2, 48000, block=480, fifo=8192)
    pos, got, rnd, ended = [0] * len(srcs), [], 0, False
    while not ended:
        if rnd == 60:
            t = L.session(srcs, 2, 48000, block=480, fifo=8192)
            t.set_state(sess.get_state())
            sess.close()
            sess = t
        blocks, eos = [], []
        for i, s in enumerate(srcs):
            total = s.pcm.size // 2
            k = min(s.rate // 100, total - pos[i])
            if i in pend and pos[i] <= pend[i][0] < pos[i] + k:
                k = pend[i][0] - pos[i]
            blocks.append(s.pcm[2 * pos[i]: 2 * (pos[i] + k)])
            eos.append(k > 0 and pos[i] + k == total)
            pos[i] += k
        sess.push_packed(blocks, eos)
        for i in [i for i in pend if pos[i] == pend[i][0]]:
            sess.push_silence(i, pend.pop(i)[1])
        while True:
            b, ended = sess.render(480)
            got.append(b)
            if b.size == 0 or ended:
                break
        rnd += 1
        assert rnd < 10000
    sess.close()
    assert not pend
    got = np.concatenate(got)
    real = [s.chain(2, 48000, s.pcm, pauses=[(2 * pauses[k][0], pauses[k][1])] if k in pauses else ()) for k, s in enumerate(srcs)]
    F.check(got, srcs, real, [s.start for s in srcs], 2, 48000, "1024 stereo sources with fades, takes and pauses")
