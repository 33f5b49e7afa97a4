"""Render time of 10 ms blocks of streaming sessions whose sources restart the mixer's conversion many times per block.
  (a) 1024 stereo 44.1 kHz decoders into a stereo 48 kHz mixer, packets of 64 to 1024 frames reported by symphonia's lagged rule and
      pushed as span marks (rb_session_push_packed_spans), 441 frames pushed and 480 rendered per block: median and p99 ms per
      render, RESTART launches per render.
  (b) 1024 stereo sources with a constant span_len of 256 samples (runs of 128 frames, shorter than a block), pushed without marks:
      a case the parent commit serves (by splitting the block into sub-blocks).  Given --parent DIR (a tree holding the parent
      commit's built rodio_b200 package), this build and that one run alternately, each in a process of its own, and must give the
      same output bytes.
Times are wall clock around the synchronised rb_session_render.  Changes no device setting; prints the card and its power limit.
    python tools/session_packet_timing.py [--parent DIR] [--blocks 200] [--warmup 20] [--rounds 3]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the card's name must come with the numbers: say why it is missing
        return f"unknown ({e})"


def packets(rng, frames):
    out, left = [], frames
    while left > 0:
        n = int(rng.choice([64, 128, 256, 576, 1024]))
        for _ in range(int(rng.integers(1, 6))):
            k = min(n, left)
            out.append(2 * k)
            left -= k
            if not left:
                break
    return out


def marks_of(pk):
    marks, start, cur = [], 0, pk[0]
    for k, n in enumerate(pk):
        if k and n != cur:
            marks.append((start + 1, n))
        cur = n if k else cur
        start += n
    return pk[0], marks


def worker(tree, case, n, blocks, warm):
    sys.path.insert(0, tree)
    import rodio_b200 as rb
    rng = np.random.default_rng(5)
    z = np.zeros(0, np.float32)
    frames = 441 * (blocks + warm + 2)
    pcm = [rng.uniform(-0.5, 0.5, 2 * frames).astype(np.float32) for _ in range(n)]
    if case == "a":
        rep = [marks_of(packets(rng, frames)) for _ in range(n)]
        spans = [r[0] for r in rep]
    else:
        rep, spans = None, [256] * n
    chains = [rb.UniformSourceIterator(rb.Source(z, 2, 44100, span_len=spans[k]), 2, 48000).low_pass(1000).amplify(0.5) for k in range(n)]
    times, launches, h = [], [], hashlib.sha256()
    with rb.Session(chains, 48000, fifo_frames=4096, max_block_frames=480, mixer_channels=2, restarts=True) as s:
        for b in range(warm + blocks):
            lo, hi = 441 * b, 441 * (b + 1)
            blk = [p[2 * lo:2 * hi] for p in pcm]
            if rep is not None:
                s.push_packed(blk, spans=[[(at - 2 * lo, sp) for at, sp in r[1] if 2 * lo <= at < 2 * hi] for r in rep])
            else:
                s.push_packed(blk)
            l0 = s.restart_launches()
            t0 = time.perf_counter()
            out, _ = s.render(480)
            t1 = time.perf_counter()
            h.update(out.tobytes())
            if b >= warm:
                times.append((t1 - t0) * 1e3)
                launches.append(s.restart_launches() - l0)
    return {"case": case, "tree": tree, "ms": times, "restart_launches": launches, "sha256": h.hexdigest()}


def run_worker(tree, case, args):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, "--case", case, "--sources", str(args.sources),
                        "--blocks", str(args.blocks), "--warmup", str(args.warmup)], capture_output=True, text=True, timeout=3000)
    if r.returncode != 0:
        raise RuntimeError(r.stdout[-2000:] + r.stderr[-3000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def summary(ms):
    a = np.asarray(ms)
    return f"median {np.median(a):.3f} ms, p99 {np.percentile(a, 99):.3f} ms, min {a.min():.3f} ms"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--sources", type=int, default=1024)
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--worker", default=None)
    ap.add_argument("--case", default="a")
    args = ap.parse_args()
    if args.worker:
        print(json.dumps(worker(args.worker, args.case, args.sources, args.blocks, args.warmup)))
        return
    print("card:", card())
    a = run_worker(ROOT, "a", args)
    la = np.asarray(a["restart_launches"])
    print(f"(a) {args.sources} stereo decoders, 10 ms blocks: {summary(a['ms'])}; RESTART launches per render: mean {la.mean():.2f}, "
          f"max {la.max()} (one class)")
    trees = [("this", ROOT)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
    got = {k: [] for k, _ in trees}
    digests = {k: set() for k, _ in trees}
    for _ in range(args.rounds):
        for k, t in trees:
            r = run_worker(t, "b", args)
            got[k] += r["ms"]
            digests[k].add(r["sha256"])
    for k, _ in trees:
        print(f"(b) span_len 256, {k} build: {summary(got[k])}")
    same = len(set().union(*digests.values())) == 1
    print("(b) output bytes identical across builds and rounds:", same)
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
