#!/usr/bin/env python
"""k_master (rb_master.cu) against k_limit_tile (rb_kernels.cu) on the same mixes, and the cfg3 render with and without
.limit(LimitSettings::mastering()) on the MixerSource.  Kernel times come from torch.profiler (CUDA activities), render
times from CUDA events on the library's stream; both after warm-up, over repeats, reported as min / median / max.  Prints
one JSON line per measurement, the card's name, power limit and maximum SM clock first."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402
import rodio_b200 as rb  # noqa: E402
from rodio_b200 import capi  # noqa: E402
from rodio_b200.source import LimitSettings, limit_effect  # noqa: E402

REPEATS = 20


def stats(v):
    v = sorted(v)
    return {"min": v[0], "median": v[len(v) // 2], "max": v[-1], "n": len(v)}


def kernel_times(pairs, repeats=REPEATS):
    """pairs: [(batch, kernel name)], rendered alternately in ONE profiler session; ms per launch of each kernel."""
    for b, _ in pairs:
        for _ in range(3):
            b.render_mix_device()
        capi.lib().rb_context_sync(b.ctx._h)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            for b, _ in pairs:
                b.render_mix_device()
                capi.lib().rb_context_sync(b.ctx._h)
    out = []
    for _, name in pairs:
        us = [e.device_time for e in prof.events() if name in e.name]
        assert len(us) == repeats, (name, len(us), sorted({e.name for e in prof.events()})[:20])
        out.append([u / 1000.0 for u in us])
    return out


def render_times(batch, repeats=REPEATS):
    import ctypes as C
    p = C.c_void_p()
    capi.check(capi.lib().rb_context_stream(batch.ctx._h, C.byref(p)), "rb_context_stream")
    st = torch.cuda.ExternalStream(p.value or 0)
    for _ in range(3):
        batch.render_mix_device()
    capi.lib().rb_context_sync(batch.ctx._h)
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        batch.render_mix_device()
        b.record(st)
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    print(json.dumps({"gpu": name, "power_limit": power, "max_sm_clock": clk}), flush=True)
    mhz = float(clk.split()[0])
    ctx = rb.default_context(0)
    torch.cuda.init()
    from test_bench_geometries_gpu import _cfg3
    srcs = _cfg3(4096, 88200)
    with rb.Batch(srcs, 1, 48000, ctx=ctx) as b:
        b.upload_all()
        cfg3_mix = b.render_mix()
        plain = render_times(b)
    with rb.Batch(srcs, 1, 48000, ctx=ctx, master=[limit_effect(LimitSettings.mastering())]) as b:
        b.upload_all()
        mastered = render_times(b)
    print(json.dumps({"case": "cfg3 render (4096 x 2 s mono, k_fused_hot)", "ms": stats(plain)}), flush=True)
    print(json.dumps({"case": "cfg3 render + MixerSource.limit(mastering)", "ms": stats(mastered)}), flush=True)
    rng = np.random.default_rng(5)
    stereo = (rng.uniform(-1, 1, 2 * 96000) * 1.5).astype(np.float32)
    for label, mix, ch in (("cfg3 mix, 96000 frames mono", cfg3_mix, 1), ("2 s stereo mix, 96000 frames", stereo, 2)):
        st = LimitSettings.mastering()
        with rb.Batch([rb.SamplesBuffer(ch, 48000, mix)], ch, 48000, flags=capi.RB_NO_FUSION, ctx=ctx, master=[limit_effect(st)]) as bn, \
                rb.Batch([rb.SamplesBuffer(ch, 48000, mix).limit(st)], ch, 48000, flags=capi.RB_NO_FUSION, ctx=ctx) as bo:
            bn.upload_all(), bo.upload_all()
            new, old = kernel_times([(bn, "k_master"), (bo, "k_limit_tile")])
            got, want = bn.render_mix(), bo.render_mix()
        frames = mix.size // ch
        med = stats(new)["median"]
        print(json.dumps({"case": label, "k_master_ms": stats(new), "k_limit_tile_ms": stats(old),
                          "k_master_cycles_per_frame_at_max_clock": round(med * 1e-3 * mhz * 1e6 / frames, 2),
                          "equal_by_value": bool(np.array_equal(got, want))}), flush=True)


if __name__ == "__main__":
    main()
