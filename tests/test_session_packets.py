"""Span reports that change as a source plays -- a decoder's packets, pushed as span marks (tests/emu/packet_scenarios.py): on the
CPU through the host-emulated library, on the H100 through the real one, bit for bit against the oracle's literal chains over a
source that reports by the same marks, summed in the documented slot order, and within 1e-5 * peak of the oracle's sequential
mixer; converter runs equal to the bootstraps of the oracle's iterator."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
sys.path[:0] = [EMU]

SCENARIOS = ["symphonia_rule", "decoder", "reports", "many_cuts", "programs", "controls", "refusals", "soak"]


@pytest.fixture(scope="module")
def hostemu(built):
    import build_emu
    return build_emu.host_lib()


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_packets_on_the_emulator(hostemu, scenario):
    r = subprocess.run([sys.executable, os.path.join(EMU, "packet_scenarios.py"), scenario], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and f"ok {scenario}" in r.stdout, (r.stdout + r.stderr)[-3000:]


@pytest.fixture(scope="module")
def packets(ctx):
    import layout_scenarios as L
    import packet_scenarios as P
    L.CTX["ctx"] = ctx
    yield P
    L.CTX["ctx"] = None


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", SCENARIOS)
def test_session_packets_on_the_device(packets, scenario):
    packets.SCENARIOS[scenario]()


@pytest.mark.gpu
def test_session_packets_at_scale(packets):
    """1024 stereo 44.1 kHz decoders with packets of 64 to 1024 frames into a 48 kHz stereo mixer, 10 ms packed pushes and renders,
    one state hand-over: bit for bit."""
    packets.scale(1024)
