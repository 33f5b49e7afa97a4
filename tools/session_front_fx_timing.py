"""Push and render time of one 10 ms block of a streaming session: 1024 stereo 44.1 kHz sources into a stereo 48 kHz mixer, with
and without a push program in front of each (fade_in(2 s).distortion(1.5, 0.9): a ramp that is still running and a clamp, so the
scatter runs both bodies for every sample).  CUDA events around the synchronised rb_session_push_packed (441 frames per source) and
around the synchronised rb_session_render (480 frames); median and min-max over the timed blocks, after warm-up.
    python tools/session_front_fx_timing.py [--sources 1024] [--blocks 200] [--warmup 20]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rodio_b200 as rb          # noqa: E402


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the card's name must come with the numbers: say why it is missing
        return f"unknown ({e})"


def time_session(n, program, blocks, warm):
    import torch
    rng = np.random.default_rng(n + program)
    z = np.zeros(0, np.float32)
    src = (lambda: rb.TestSource(z, 2, 44100).fade_in(2_000_000_000).distortion(1.5, 0.9)) if program else (lambda: rb.TestSource(z, 2, 44100))
    chains = [rb.UniformSourceIterator(src(), 2, 48000).low_pass(1000).amplify(0.5) for _ in range(n)]
    block = list(rng.uniform(-0.5, 0.5, (n, 441 * 2)).astype(np.float32))
    t_push, t_render = [], []
    with rb.Session(chains, 48000, fifo_frames=4096, max_block_frames=480, mixer_channels=2) as s:
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for k in range(warm + blocks):
            torch.cuda.synchronize()
            ev[0].record()
            s.push_packed(block)
            ev[1].record()
            out, _ = s.render(480)
            ev[2].record()
            torch.cuda.synchronize()
            assert out.size > 0
            if k >= warm:
                t_push.append(ev[0].elapsed_time(ev[1]))
                t_render.append(ev[1].elapsed_time(ev[2]))
    return [(np.median(t), np.min(t), np.max(t)) for t in (t_push, t_render)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    print("card:", card())
    for program in (False, True, False, True):     # alternated: the spread between repeats is part of the result
        (pm, plo, phi), (rm, rlo, rhi) = time_session(a.sources, program, a.blocks, a.warmup)
        print(f"{a.sources} stereo sources, {'with' if program else 'without'} a program: push median {pm:.3f} ms (min {plo:.3f}, max {phi:.3f}); "
              f"render median {rm:.3f} ms (min {rlo:.3f}, max {rhi:.3f})", flush=True)


if __name__ == "__main__":
    main()
