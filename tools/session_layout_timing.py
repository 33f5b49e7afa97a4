"""Render time of one 10 ms block of a streaming session: N 5.1 sources (44.1 kHz, low_pass + amplify) into a 6-channel 48 kHz
mixer, against the same N stereo sources into a stereo mixer.  CUDA events around synchronised rb_session_render calls, after
warm-up; every block is pushed (packed, 441 frames per source) before it is rendered, outside the timed window.
    python tools/session_layout_timing.py [--sources 256 1024] [--blocks 200]"""
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


def time_session(n, ch, blocks, warm):
    import torch
    rng = np.random.default_rng(n * 10 + ch)
    chains = [rb.UniformSourceIterator(rb.TestSource(np.zeros(0, np.float32), ch, 44100), ch, 48000).low_pass(1000).amplify(0.5)
              for _ in range(n)]
    block = (rng.uniform(-0.5, 0.5, (n, 441 * ch)).astype(np.float32))
    times = []
    with rb.Session(chains, 48000, fifo_frames=4096, max_block_frames=480, mixer_channels=ch) as s:
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for k in range(warm + blocks):
            s.push_packed(list(block))
            torch.cuda.synchronize()
            start.record()
            out, _ = s.render(480)
            stop.record()
            torch.cuda.synchronize()
            if k >= warm:
                times.append(start.elapsed_time(stop))
            assert out.size > 0
    return np.median(times), np.min(times), np.max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, nargs="+", default=[256, 1024])
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    print("card:", card())
    for n in a.sources:
        for ch, what in ((6, "5.1 -> 6-ch mixer"), (2, "stereo -> stereo mixer")):
            med, lo, hi = time_session(n, ch, a.blocks, a.warmup)
            print(f"{n:5d} sources, {what:22s}: render of 10 ms  median {med:.3f} ms  (min {lo:.3f}, max {hi:.3f})", flush=True)


if __name__ == "__main__":
    main()
