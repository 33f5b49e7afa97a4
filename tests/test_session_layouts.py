"""Streaming sessions of up to 12 channels, with sources of any channel count (tests/emu/layout_scenarios.py): on the CPU through
the host-emulated library, on the H100 through the real one -- bit for bit against the oracle's chains summed in the documented slot
order, and within 1e-5 * peak of the oracle's sequential mixer."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
sys.path[:0] = [EMU]

CPU_SCENARIOS = ["layout_matrix", "mixed_layouts_hand_over", "chain_variants", "split_invariance", "controls", "volume_changes",
                 "today_shapes_blob", "coverage", "refusals", "fifo_errors"]


@pytest.fixture(scope="module")
def hostemu(built):
    import build_emu
    return build_emu.host_lib()


@pytest.mark.parametrize("scenario", CPU_SCENARIOS)
def test_session_layouts_on_the_emulator(hostemu, scenario):
    r = subprocess.run([sys.executable, os.path.join(EMU, "layout_scenarios.py"), scenario], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and f"ok {scenario}" in r.stdout, (r.stdout + r.stderr)[-3000:]


@pytest.fixture(scope="module")
def layouts(ctx):
    import layout_scenarios as L
    L.CTX["ctx"] = ctx
    yield L
    L.CTX["ctx"] = None


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", [s for s in CPU_SCENARIOS if s != "coverage"])
def test_session_layouts_on_the_device(layouts, scenario):
    layouts.SCENARIOS[scenario]()


@pytest.mark.gpu
def test_session_51_at_scale(layouts):
    """1024 5.1 sources at 44.1 kHz into a 6-channel 48 kHz mixer, 10 ms packed pushes and renders over 2 s, one state hand-over."""
    L = layouts
    srcs = [L.Src(6, 44100, start=0 if k % 5 else 3 * k, frames=88200 - 17 * k, seed=20000 + k) for k in range(1024)]
    L.run_case(srcs, 6, 48000, 3, "1024 5.1 sources", hand_over=100, split=False)


@pytest.mark.gpu
def test_session_6ch_with_limiter(layouts, ctx):
    """mixer_source.limit(LimitSettings::mastering()) on a 6-channel session equals k_limit_tile over the unlimited session output."""
    import rodio_b200 as rb
    from rodio_b200 import capi
    from rodio_b200.source import LimitSettings, limit_effect
    L = layouts
    srcs = [L.Src(ci, r, frames=9000 + 13 * k, gain=2.5, seed=21000 + k)
            for k, (ci, r) in enumerate([(6, 44100), (2, 48000), (1, 22050), (8, 96000), (6, 48000), (3, 44100)] * 6)]
    outs = []
    for master in ((), (limit_effect(LimitSettings.mastering()),)):
        s = L.session(srcs, 6, 48000, block=480, master=master)
        got, s = L.drive(s, srcs, np.random.default_rng(8), [r.rate // 100 for r in srcs], 480, split=False)
        s.close()
        outs.append(got)
    assert outs[0].size == outs[1].size and float(np.max(np.abs(outs[0]))) > 1.0   # every source starts at 0: no gaps; loud enough to limit
    with rb.Batch([rb.SamplesBuffer(6, 48000, outs[0]).limit(LimitSettings.mastering())], 6, 48000, flags=capi.RB_NO_FUSION, ctx=ctx) as b:
        b.upload_all()
        want = b.render_mix()
    assert np.array_equal(outs[1], want), "6-channel session behind the limiter != k_limit_tile over its unlimited output"
