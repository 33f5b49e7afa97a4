"""Render time of streaming sessions whose sources are generators (RB_FX_SIGNAL: the session fills their FIFOs on the device), beside
the same sessions fed the same samples from the host by rb_session_push_packed, which is what a caller did without generator sources.
  (a) BASELINE cfg2 live: 1024 SineWaves into mixer(1, 48000), 480-frame blocks.
  (b) 4096 SineWaves at 48 kHz, take_duration(1 s), into a stereo 44.1 kHz mixer with RB_SESSION_RESTARTS, 441-frame blocks (the twin
      gets 480 frames per source and block).
The two sessions of a case render alternately, block by block, on one context; both must give the same bytes where both rendered.  Times are wall clock
around the synchronised calls: rb_session_render of the generator session; rb_session_push_packed and rb_session_render of the twin.
Changes no device setting; prints the card and its power limit.
    python tools/session_generator_timing.py [--blocks 200] [--warmup 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the card's name must come with the numbers: say why it is missing
        return f"unknown ({e})"


def summary(ms):
    a = np.asarray(ms)
    return f"median {np.median(a):.3f} ms, p99 {np.percentile(a, 99):.3f} ms, min {a.min():.3f} ms"


def run(name, gens, mix_ch, mix_rate, block, push, blocks, warm, restarts):
    import oracle
    import rodio_b200 as rb
    n = len(gens)
    total = push * (blocks + warm + 2)
    pcm = [oracle.signal(g.function, g.rate, g.frequency, total) for g, _ in gens]
    gen_chains = [rb.UniformSourceIterator(prog(g), mix_ch, mix_rate) for g, prog in gens]
    twin_chains = [rb.UniformSourceIterator(prog(rb.TestSource(np.zeros(0, np.float32), 1, g.rate)), mix_ch, mix_rate) for g, prog in gens]
    kw = dict(fifo_frames=4096, max_block_frames=block, mixer_channels=mix_ch, restarts=restarts)
    t_gen, t_push, t_render, og, ot = [], [], [], [], []
    with rb.Session(gen_chains, mix_rate, **kw) as sg, rb.Session(twin_chains, mix_rate, **kw) as st:
        for b in range(warm + blocks):
            t0 = time.perf_counter()
            a, _ = sg.render(block)
            t1 = time.perf_counter()
            st.push_packed([p[push * b: push * (b + 1)] for p in pcm])
            t2 = time.perf_counter()
            c, _ = st.render(block)
            t3 = time.perf_counter()
            og.append(a), ot.append(c)
            if b >= warm:
                t_gen.append((t1 - t0) * 1e3), t_push.append((t2 - t1) * 1e3), t_render.append((t3 - t2) * 1e3)
    print(f"{name}: {n} sources, {blocks} blocks of {block} frames")
    print(f"  generator session, rb_session_render:        {summary(t_gen)}")
    print(f"  pushed twin, rb_session_push_packed:         {summary(t_push)}")
    print(f"  pushed twin, rb_session_render:              {summary(t_render)}")
    print(f"  pushed twin, push_packed + render:           {summary(np.asarray(t_push) + np.asarray(t_render))}")
    og, ot = np.concatenate(og), np.concatenate(ot)   # the twin may trail by the frame whose right neighbour it has not got yet
    k = min(og.size, ot.size)
    same = k > 0 and np.array_equal(og[:k].view(np.uint32), ot[:k].view(np.uint32))
    print(f"  output bytes identical over the {k // mix_ch} frames both rendered: {same}")
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import rodio_b200 as rb
    print("card:", card())
    freqs = lambda n: [min(110.0 * 2.0 ** (s / 128.0), 19999.0) for s in range(n)]
    ok = run("(a) cfg2 live mixer", [(rb.SineWave(f), lambda s: s) for f in freqs(1024)], 1, 48000, 480, 480, args.blocks, args.warmup, False)
    d = rb.Duration.from_secs(1)
    # 1 s takes: 100 blocks of 441 frames play them out; the timed window stays inside them
    blocks = min(args.blocks, 100 - args.warmup - 2)
    ok &= run("(b) resampled 1 s takes with restarts", [(rb.SineWave(f), lambda s: s.amplify(0.1).take_duration(d)) for f in freqs(4096)],
              2, 44100, 441, 480, blocks, args.warmup, True)
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
