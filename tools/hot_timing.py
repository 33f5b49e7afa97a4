#!/usr/bin/env python
"""Where does a tile iteration of k_fused_hot go?  Builds an instrumented copy of the library
(-DRB_HOT_TIMING: clock64 around each warp's work and its wait at the tile barrier), runs the bench
workload once and prints, per warp, the share of cycles spent working vs waiting.  Diagnostic only.
--ablate-smem: the full kernel, conflict-free window addresses (bit 16) and no stage-A t stores (bit 64), three
renders each in turn, to bound what stage A's shared-memory traffic costs."""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "rodio_b200", "librodio_b200_timing.so")
if "--build-only" in sys.argv or not os.path.exists(LIB):
    from rodio_b200 import build
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    build.build(force=True, extra_flags=["-DRB_HOT_TIMING"], out=LIB)
    if "--build-only" in sys.argv:
        sys.exit(0)
os.environ["RODIO_B200_LIB"] = LIB

import numpy as np  # noqa: E402
import torch  # noqa: E402
import rodio_b200 as rb  # noqa: E402
from rodio_b200 import dist as rbd  # noqa: E402


def main():
    S = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 4096
    ch = 2 if "--stereo" in sys.argv else 1
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("gpu:", q.stdout.strip() or q.stderr.strip())
    ctx = rb.default_context(0)
    dev = torch.device("cuda", 0)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream, device=dev)
    z = np.zeros(44100 * 2 * ch, np.float32)
    srcs = [rb.UniformSourceIterator(rb.TestSource(z, ch, 44100), ch, 48000).low_pass(200).amplify(1.2) for _ in range(S)]
    lib = C.CDLL(LIB)
    buf = (C.c_ulonglong * 128)()
    with rb.Batch(srcs, ch, 48000, ctx=ctx) as b:
        for i in range(S):
            p, cap = b.input_device_ptr(i)
            with torch.cuda.stream(ext):
                torch.as_tensor(rbd.DeviceArray(p, cap), device=dev).uniform_(-0.5, 0.5)
        for _ in range(3):
            b.render_mix_device()
        torch.cuda.synchronize()
        skips = [0, 1, 2, 4, 8, 1 | 4 | 8, 2 | 4, 1 | 2 | 4] if "--skips" in sys.argv else [0]
        if "--ablate" in sys.argv:
            skips = [0, 1 | 4 | 8, 2 | 4, 2]
        if "--ablate-smem" in sys.argv:
            skips = [0, 16, 64] * 3
        names = {1: "no stage A", 2: "no recurrence", 4: "no stage C", 8: "no second rows", 16: "conflict-free window reads", 32: "no range check",
                 64: "no stage-A t stores"}
        for skip in skips:
            lib.rb_debug_hot_skip(skip)
            lib.rb_debug_hot_timing(buf, 1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            b.render_mix_device()
            e1.record(ext)
            torch.cuda.synchronize()
            lib.rb_debug_hot_timing(buf, 0)
            ms = e0.elapsed_time(e1)
            what = " + ".join(v for k, v in names.items() if skip & k) or "full kernel"
            print(json.dumps({"streams": S, "channels": ch, "ms": round(ms, 4), "variant": what}))
            # warp roles of k_fused_hot at 32 rows per CTA (rb_fused.cu: hot_row_slot / hot_first_row / hot_second_row, stage C
            # on slots 6, 7); with fewer rows per CTA the later warps of a group own fewer rows or none
            groups = {"two rows (w0,1,2,4,5,6,10,12,13,16,17)": [0, 1, 2, 4, 5, 6, 10, 12, 13, 16, 17], "stage C (w8,9)": [8, 9],
                      "one row": [14, 18, 20, 21, 22, 24, 25, 26, 28, 29], "loader": [30],
                      "recurrence": [31] + ([27] if ch == 2 else [])}
            n_cta = int(b.mix_group and (S + b.mix_group - 1) // b.mix_group) or 1
            for g, ws in groups.items():
                work = sum(buf[4 * w] for w in ws) / len(ws) / n_cta
                bar = sum(buf[4 * w + 1] for w in ws) / len(ws) / n_cta
                mwait = sum(buf[4 * w + 2] for w in ws) / len(ws) / n_cta
                print(f"    {g:22s} work {work / 1e6:6.3f} Mcycles (of which window wait {mwait / 1e6:6.3f})  barrier {bar / 1e6:6.3f} Mcycles")


if __name__ == "__main__":
    main()
