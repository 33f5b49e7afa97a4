"""Generator sources in streaming sessions (tests/emu/generator_scenarios.py): SineWave / SignalGenerator chains generated into the
FIFOs by the session itself, on the CPU through the host-emulated library and on the H100 through the real one, bit for bit against
the same sessions fed the oracle's generator samples by pushes, and against the oracle's chains summed in the documented slot order."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
sys.path[:0] = [EMU]

SCENARIOS = ["equivalence", "examples", "controls", "state", "soak", "errors"]


@pytest.fixture(scope="module")
def hostemu(built):
    import build_emu
    return build_emu.host_lib()


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_generators_on_the_emulator(hostemu, scenario):
    r = subprocess.run([sys.executable, os.path.join(EMU, "generator_scenarios.py"), scenario], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and f"ok {scenario}" in r.stdout, (r.stdout + r.stderr)[-3000:]


def test_signal_generator_adapters_read_like_rodio(built):
    """SineWave(740.0).amplify(0.1).take_duration(d): the adapters apply to the endless generator; .take(n) is unchanged."""
    import rodio_b200 as rb
    from rodio_b200 import _capi as capi
    s = rb.SineWave(740.0).amplify(0.1).take_duration(rb.Duration.from_secs(1))
    assert [e.kind for e in s.effects] == [capi.RB_FX_SIGNAL, capi.RB_FX_AMPLIFY, capi.RB_FX_TAKE_DURATION]
    assert s.effects[0].ns[0] == 2**64 - 1 and s.effects[0].f32[0] == np.float32(740.0) and s.sample_rate() == 48000
    assert rb.SineWave(440.0).take(100).effects[0].ns[0] == 100
    u = rb.UniformSourceIterator(rb.SquareWave(440.0), 2, 44100)
    assert [e.kind for e in u.effects] == [capi.RB_FX_SIGNAL, capi.RB_FX_UNIFORM] and u.effects[0].u32[0] == capi.RB_SIGNAL_SQUARE
    with pytest.raises(AttributeError):
        rb.SineWave(440.0).no_such_adapter


@pytest.fixture(scope="module")
def gen_scenarios(ctx):
    import layout_scenarios as L
    import generator_scenarios as G
    L.CTX["ctx"] = ctx
    yield G
    L.CTX["ctx"] = None


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_generators_on_the_device(gen_scenarios, scenario):
    gen_scenarios.SCENARIOS[scenario]()


def cfg2_frequencies(n):
    return [min(110.0 * 2.0 ** (s / 128.0), 19999.0) for s in range(n)]


@pytest.mark.gpu
def test_session_1024_sines_against_pushed_twin(gen_scenarios):
    """BASELINE cfg2 as a live mixer: 1024 SineWaves into mixer(1, 48000), 2 s in 480-frame blocks."""
    G = gen_scenarios
    srcs = [G.GSrc(48000, f, lp=None, gain=None, seed=k) for k, f in enumerate(cfg2_frequencies(1024))]
    frames = 2 * 48000
    gen, twin, _ = G.sessions(srcs, 1, 48000, block=480, fifo=4096, out_frames=frames)
    got, ref = [], []
    for _ in range(frames // 480):
        a, _ = gen.render(480)
        b, _ = twin.render(480)
        assert a.size == 480
        got.append(a), ref.append(b)
    G.assert_bit_exact(np.concatenate(got), np.concatenate(ref), "1024 sines")
    gen.close(), twin.close()


@pytest.mark.gpu
def test_session_4096_resampled_takes_against_pushed_twin(gen_scenarios):
    """4096 SineWaves at 48 kHz with take_duration(1 s) into a stereo 44.1 kHz mixer with RB_SESSION_RESTARTS: two converter runs
    each, the same bytes and run counts as the pushed twin."""
    G = gen_scenarios
    srcs = [G.GSrc(48000, f, prog=[("amp", 0.1), ("take", 1000 * G.MS, False)], lp=None, gain=None, seed=k)
            for k, f in enumerate(cfg2_frequencies(4096))]
    gen, twin, _ = G.sessions(srcs, 2, 44100, block=441, fifo=4096, restarts=True)
    got, ref, ended = [], [], False
    while not ended:
        a, ended = gen.render(441)
        b, e2 = twin.render(441)
        assert a.size == b.size and ended == e2
        got.append(a), ref.append(b)
        assert len(got) < 1000
    G.assert_bit_exact(np.concatenate(got), np.concatenate(ref), "4096 resampled takes")
    assert all(gen.source_runs(i) == twin.source_runs(i) == 2 for i in range(0, 4096, 97))
    gen.close(), twin.close()
