"""Render time of one 10 ms block of a streaming session with restart schedules (RB_SESSION_RESTARTS): 1024 stereo 44.1 kHz sources
into a stereo 48 kHz mixer, low_pass + amplify behind the conversion, 441 frames pushed and 480 rendered per block.  Three sessions,
alternated twice: without the flag (span_len ignored); with it and span_len = 32768 for every source (all sources restart in the
same block, every 37th or so); with it and span_len staggered from source to source (some source restarts in every block).  CUDA
events around the synchronised rb_session_render; median and min-max over the timed blocks after warm-up, the blocks that launched
a RESTART kernel and the others apart.  Changes no device setting; prints the card, its power limit and its clocks with the numbers.
    python tools/session_restart_timing.py [--sources 1024] [--blocks 200] [--warmup 20]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rodio_b200 as rb          # noqa: E402


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the card's name must come with the numbers: say why it is missing
        return f"unknown ({e})"


def time_session(n, mode, blocks, warm):
    import torch
    rng = np.random.default_rng(n)
    z = np.zeros(0, np.float32)
    span = {"off": lambda k: 32768, "aligned": lambda k: 32768, "staggered": lambda k: 2 * (8000 + 16 * (k % 512))}[mode]
    chains = [rb.UniformSourceIterator(rb.Source(z, 2, 44100, span_len=span(k)), 2, 48000).low_pass(1000).amplify(0.5) for k in range(n)]
    block = list(rng.uniform(-0.5, 0.5, (n, 441 * 2)).astype(np.float32))
    with_cut, without = [], []
    with rb.Session(chains, 48000, fifo_frames=4096, max_block_frames=480, mixer_channels=2, restarts=mode != "off") as s:
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for k in range(warm + blocks):
            s.push_packed(block)
            before = s.restart_launches()
            torch.cuda.synchronize()
            ev[0].record()
            out, _ = s.render(480)
            ev[1].record()
            torch.cuda.synchronize()
            assert out.size > 0
            if k >= warm:
                (with_cut if s.restart_launches() > before else without).append(ev[0].elapsed_time(ev[1]))
        runs = s.source_runs(0)
    return with_cut, without, runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    print("card (name, power limit, max SM clock, SM clock now):", card())
    fmt = lambda t: f"{len(t)} blocks, median {np.median(t):.3f} ms (min {np.min(t):.3f}, max {np.max(t):.3f})" if t else "0 blocks"
    for mode in ("off", "aligned", "staggered") * 2:     # alternated: the spread between repeats is part of the result
        with_cut, without, runs = time_session(a.sources, mode, a.blocks, a.warmup)
        print(f"{a.sources} stereo sources, restarts {mode}: render without a restart: {fmt(without)}; with a RESTART launch: {fmt(with_cut)}; "
              f"source 0 started {runs} runs", flush=True)


if __name__ == "__main__":
    main()
