"""Restart schedules in streaming sessions -- the mixer's conversion restarted where rodio's UniformSourceIterator restarts it, for
sources that report spans and behind take_duration (tests/emu/restart_scenarios.py): on the CPU through the host-emulated library,
on the H100 through the real one, bit for bit against the oracle's chains summed in the documented slot order and within
1e-5 * peak of the oracle's sequential mixer."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
sys.path[:0] = [EMU]

SCENARIOS = ["spans", "takes", "split_invariance", "controls", "refusals", "soak"]


@pytest.fixture(scope="module")
def hostemu(built):
    import build_emu
    return build_emu.host_lib()


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_restarts_on_the_emulator(hostemu, scenario):
    r = subprocess.run([sys.executable, os.path.join(EMU, "restart_scenarios.py"), scenario], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and f"ok {scenario}" in r.stdout, (r.stdout + r.stderr)[-3000:]


@pytest.fixture(scope="module")
def restarts(ctx):
    import layout_scenarios as L
    import restart_scenarios as R
    L.CTX["ctx"] = ctx
    yield R
    L.CTX["ctx"] = None


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_restarts_on_the_device(restarts, scenario):
    restarts.SCENARIOS[scenario]()


@pytest.mark.gpu
def test_session_restarts_at_scale(restarts):
    """1024 stereo 44.1 kHz sources into a 48 kHz stereo mixer, each fade_in(200 ms).take_duration(1.5 s) with the fade-out filter: five
    converter runs per source, more where a pause ends a run early (a tenth of the sources); 10 ms packed pushes and renders, one
    state hand-over."""
    R = restarts
    F = R.F
    take = 2 * 66150
    srcs = [R.RSrc(2, 44100, [("fade_in", 200 * R.MS), R.take_of(44100, 2, take)], kind="pre", pre=1.0, lp=None if k % 3 else 700,
                   frames=70560 - 7 * (k % 50), start=0 if k % 7 else 3 * k, seed=40000 + k) for k in range(1024)]
    pauses = [[(4800 + 37 * (k % 11), 2400 + k)] if k % 10 == 0 else [] for k in range(1024)]
    sess = R.session(srcs, 2, 48000, block=480, fifo=8192)
    got, sess = R.drive(sess, srcs, block=480, pauses=pauses, hooks={60: R.hand_over(srcs, 2, 48000, block=480, fifo=8192)})
    runs = [sess.source_runs(i) for i in range(1024)]
    launches = sess.restart_launches()
    sess.close()
    assert all(r == 5 for k, r in enumerate(runs) if k % 10) and all(r >= 5 for r in runs) and launches > 0, (runs[:12], launches)
    real = [s.chain(2, 48000, s.pcm, pauses=[(2 * at, n) for at, n in p]) for s, p in zip(srcs, pauses)]
    F.check(got, srcs, real, [s.start for s in srcs], 2, 48000, "1024 stereo sources with takes of five runs and pauses")
