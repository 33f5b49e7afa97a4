// rb_session_plan.h — host-side bookkeeping of a streaming session (plain C++, no CUDA): which mixer frames the next
// render can produce from the PCM pushed so far, which part of every stream's FIFO the block reads, and what is left
// for the next block.  Shared by rb_session.cu and by the CPU emulator under tests/emu/, so the whole block logic is
// exercised on the CPU against whole-stream renders.
//
// What it replaces: rodio pulls one sample at a time through MixerSource::next (src/mixer.rs:120-136) ->
// UniformSourceIterator::next (src/source/uniform.rs:78-97) -> SampleRateConverter::next
// (src/conversions/sample_rate.rs:131-201); every adapter keeps its state between calls.  A block render must carry
// exactly that state from block to block:
//   * resampler: the stream-absolute index of the next output frame (its numerator and left frame follow from it:
//     (o * from) mod to and floor(o * from / to)) and the input frames from that left frame on -- they stay in the
//     stream's FIFO; an output is only rendered once its right neighbour has arrived, or the stream has ended (the
//     last frame is then emitted raw, sample_rate.rs:187-199);
//   * biquad: x[n-1], x[n-2], y[n-1], y[n-2] (src/source/blt.rs:397-410) -- four floats per stream on the device; a filter
//     in FRONT of the conversion additionally has a position of its own in the input (Stream::fpos): it has consumed the
//     right neighbour of the last output already, so its two last outputs are the interpolation taps.
//   * restarts (RB_SESSION_RESTARTS): UniformSourceIterator does not convert a source as one run.  At every bootstrap it asks
//     current_span_len(), caps it at 32768 samples and builds a fresh SampleRateConverter over that many samples
//     (src/source/uniform.rs:50-68, :83-96); the run pulls its first two frames at once, interpolates inside itself only and emits
//     its last frame raw.  A stream with a schedule keeps the run the next output belongs to -- its first input and output frame --
//     and the ends of the runs the pushes have begun; everything above applies to each run with indices relative to its start.
//     What the source reports may change as it plays (a decoder reports the length of the packet it decoded last,
//     src/decoder/symphonia.rs:199-201): the pushes carry those changes, and every bootstrap a push begins takes the report in
//     effect at its position.  A run's end is fixed when it begins, so the only state is the report at the pushed end.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace session {

struct Stream {
    uint32_t from = 1, to = 1; // the source's rate pair, reduced (from <= to; 1:1 = already at the mixer's rate)
    uint64_t mix_start = 0;    // mixer frame the stream joins at (frame aligned, src/mixer.rs:175-183)
    uint64_t pushed = 0;       // input frames received so far
    uint64_t out_done = 0;     // output frames rendered so far (= stream-absolute index of the next one)
    uint64_t i0 = 0;           // stream-absolute index of the frame at the front of the FIFO (multiple of 4)
    bool eof = false;          // no more input will come
    bool held = false;         // declared when the session was created but not handed to the mixer yet (Mixer::add comes
                               // later): it takes pushes, renders nothing and holds nobody up until it is started
    int64_t follows = -1;      // held source that starts on the frame after source `follows` has played out -- the
                               // sources of a queue (src/queue.rs:128-192: the next sound begins where the current one ends)
    uint64_t fpos = 0;         // input frames [0, fpos) have been pulled by the converter (stream-absolute): up to the right
                               // neighbour of the last output -- a gain in front of the conversion is final for them
    bool front = false;        // the source's filter sits in front of the conversion, runs once per INPUT frame and has
                               // consumed exactly those frames: the FIFO must keep everything from fpos on
    // ---- restart schedule; run_cap == 0: none, the source is one run (every session without RB_SESSION_RESTARTS) ----
    uint64_t run_cap = 0;      // frames a run that begins now holds at most, from the report in effect at the pushed end:
                               // min(report, 32768) samples; NO_LIMIT: None (the run lasts as long as the source); BAD_CAP: a
                               // report no run may begin under (not whole frames, or under two)
    uint64_t run_i = 0;        // the run of output `out_done`: its first input frame ...
    uint64_t run_o = 0;        // ... and its first output frame (stream-absolute)
    uint64_t sched_end = 0;    // input frame at which the run the pushes are filling ends (0: nothing pushed yet)
    uint64_t runs_done = 0;    // runs played out
    std::vector<uint64_t> ends;   // ends (input frame) of the runs begun by a push and not played out: ends[0] is the current run's
    uint64_t fill() const { return pushed - i0; }   // frames in the FIFO
};

// SampleRateConverter output length for L input frames on the reduced grid from:to, from != to
// (closed form of src/conversions/sample_rate.rs:157-199; rb_sample_rate_out_len in the C ABI is the same formula).
inline uint64_t out_total(uint64_t L, uint32_t from, uint32_t to) {
    if (L == 0) return 0;
    if (L == 1) return 1;
    const uint64_t ns = ((L - 1) * (uint64_t)to + from - 1) / from;   // first output whose left frame is L-1
    return ns + ((ns * (uint64_t)from < L * (uint64_t)to) ? 1 : 0);
}
// Outputs [0, n) whose right neighbour exists among L frames: n = ceil((L-1) * to / from).
inline uint64_t out_interp(uint64_t L, uint32_t from, uint32_t to) {
    return L < 2 ? 0 : ((L - 1) * (uint64_t)to + from - 1) / from;
}
constexpr uint64_t NO_LIMIT = ~0ull;       // run_cap: the source reports None (and no take limits it)
constexpr uint64_t BAD_CAP = ~0ull - 1;    // run_cap: a run may not begin under the report in effect
// A change of what the source reports, inside a push: bootstraps from frame `at` of the push on begin runs of at most `cap` frames.
struct CapChange {
    uint64_t at, cap;
};
// A push of n frames (PCM, or a pause's silence: real = false) is about to move `pushed`: the runs whose first frame is among
// them begin.  A run's length is known when it begins -- run_cap, or what the source's take still lets through at that moment
// (take_left frames, ~0: no take; src/source/take.rs:180-196), the silence inside the run counted against it as rodio's Take
// counts Pausable's zeros.  changes[0 .. n_changes) (increasing `at`) move run_cap as the push goes: a bootstrap at frame k of the
// push sees those with at <= k; run_cap ends as the push leaves it.  A stream without a schedule only takes one when its first
// bootstrap -- frame 0 of its first push -- sees a limit.  Returns false, having changed nothing, when a run would begin under
// BAD_CAP.
inline bool schedule_push(Stream& s, uint64_t n, uint64_t take_left, bool real, const CapChange* changes = nullptr, size_t n_changes = 0) {
    size_t c = 0;
    auto apply = [&](uint64_t k) {
        for (; c < n_changes && changes[c].at <= k; c++) s.run_cap = changes[c].cap;
    };
    if (!s.run_cap) {
        if (s.pushed || !n_changes || changes[0].at || n == 0) return true;
        const Stream keep = s;
        apply(0);
        if (s.run_cap == NO_LIMIT) s.run_cap = 0;   // None at the first bootstrap: one run for good
        if (!s.run_cap) return true;
        if (!schedule_push(s, n, take_left, real, changes + c, n_changes - c)) return s = keep, false;
        return true;
    }
    const Stream keep = s;
    for (uint64_t at = s.pushed, stop = s.pushed + n; at < stop;) {
        if (at == s.sched_end) {
            apply(at - s.pushed);
            if (s.run_cap == BAD_CAP) return s = keep, false;
            const uint64_t len = std::min(s.run_cap, take_left);
            s.sched_end = len >= NO_LIMIT - at ? NO_LIMIT : at + len, s.ends.push_back(s.sched_end);
        }
        const uint64_t step = std::min(stop, s.sched_end) - at;
        if (real && take_left != ~0ull) take_left -= step;
        at += step;
    }
    apply(NO_LIMIT);
    return true;
}
// Output frames of stream `s` that exist so far (renderable): everything once it has ended, else the interpolated ones.  With a
// schedule, run by run: a run whose last frame has arrived is complete, its raw last frame included, whatever follows.
inline uint64_t out_ready(const Stream& s) {
    if (!s.run_cap) return s.eof ? out_total(s.pushed, s.from, s.to) : out_interp(s.pushed, s.from, s.to);
    uint64_t i = s.run_i, o = s.run_o;
    for (uint64_t e : s.ends) {
        const uint64_t L = std::min(s.pushed, e) - i;
        if (s.pushed < e && !s.eof) return o + out_interp(L, s.from, s.to);
        o += out_total(L, s.from, s.to), i = e;
    }
    return o;
}
// All of the stream's output frames, once it has its end of stream.
inline uint64_t out_end(const Stream& s) { return s.run_cap ? out_ready(s) : out_total(s.pushed, s.from, s.to); }
inline bool finished(const Stream& s) { return s.eof && s.out_done >= out_end(s); }
// Moves to the run of output `out_done`: runs that are complete and played out are left behind.
inline void settle(Stream& s) {
    while (!s.ends.empty() && (s.pushed >= s.ends[0] || s.eof)) {
        const uint64_t e = std::min(s.pushed, s.ends[0]), n = out_total(e - s.run_i, s.from, s.to);
        if (s.out_done < s.run_o + n) break;
        s.run_i = e, s.run_o += n, s.runs_done++;
        s.ends.erase(s.ends.begin());
    }
}
// Converter runs that have produced an output so far.
inline uint64_t runs_started(const Stream& s) { return s.runs_done + (s.out_done > s.run_o ? 1 : 0); }

// How many mixer frames [T, T + n) can be rendered now (every unfinished stream must be able to supply its part).
// Returns 0 with *ended = true when no stream is left (MixerSource::next returns None, src/mixer.rs:129-135).
// A queued source can be scheduled as soon as the end of its predecessor is known, i.e. once that one has received all
// of its input: its first frame follows the predecessor's last.  (Chains resolve front to back.)
// A predecessor that has played out before the successor was queued (Player::append on a player whose queue has run dry:
// the sound starts at the current position) hands over at T, the frame rendered next -- never behind the timeline, where the
// successor could neither render its head nor let the session move on.
inline void resolve_queue(std::vector<Stream>& st, uint64_t T) {
    for (bool again = true; again;) {
        again = false;
        for (Stream& s : st) {
            if (!s.held || s.follows < 0) continue;
            const Stream& p = st[(size_t)s.follows];
            if (p.held || !p.eof) continue;
            s.mix_start = std::max(T, p.mix_start + out_end(p));
            s.held = false, again = true;
        }
    }
}

inline uint64_t renderable(const std::vector<Stream>& st, uint64_t T, uint64_t max_frames, bool* ended) {
    uint64_t n = max_frames;
    bool active = false, waiting = false;
    for (const Stream& s : st) {
        if (s.held) {             // may still be added: keeps the session alive, holds nobody up
            waiting = true;
            continue;
        }
        if (finished(s)) continue;
        active = true;
        const uint64_t upto = s.mix_start + out_ready(s);   // the stream can cover the timeline up to here
        n = std::min(n, upto > T ? upto - T : 0);
    }
    *ended = !active && !waiting;
    return active ? n : 0;        // nothing is playing: MixerSource::next() is None, the timeline stands still (mixer.rs:129-135)
}

// A restart inside a block: outputs from block-local m on belong to the run that begins at input frame i, has frames up to `end`
// so far and interpolates on its first n_int outputs (of those in the block)
struct RunCut {
    uint64_t m, i, end, n_int;
};
// One stream's part of the block [T, T + n).
struct Part {
    uint64_t mix_start = 0;   // block-local timeline position of its first output
    uint64_t out_len = 0;     // outputs it contributes
    uint64_t o0 = 0;          // index of the first of them in its converter run (stream-absolute without a schedule)
    uint64_t n_int = 0;       // how many of them interpolate (the rest is the raw last frame); with cuts: of those in front of the first
    bool continues = false;   // more outputs will follow in later blocks
    uint64_t o_abs = 0;       // stream-absolute index of the first output
    uint64_t run_i = 0;       // first input frame of the run of o0 (stream-absolute) ...
    uint64_t run_end = 0;     // ... and the frame behind the last one of it that has arrived
    std::vector<RunCut> cuts;  // the block's restarts, in order: any number of runs may begin inside it
};
// (after settle)
inline Part part_of(const Stream& s, uint64_t T, uint64_t n) {
    Part p;
    if (s.held) {
        p.continues = true;
        return p;
    }
    const uint32_t from = s.from, to = s.to;
    const uint64_t ready = out_ready(s);
    const uint64_t lo = std::max(T, s.mix_start + s.out_done), hi = std::min(T + n, s.mix_start + ready);
    if (lo >= hi) {
        p.continues = !finished(s);
        return p;
    }
    p.mix_start = lo - T, p.out_len = hi - lo, p.o_abs = lo - s.mix_start;
    p.run_i = s.run_i, p.run_end = s.run_cap ? std::min(s.pushed, s.ends[0]) : s.pushed;
    p.o0 = p.o_abs - s.run_o;
    const uint64_t ni = out_interp(p.run_end - p.run_i, from, to);
    p.n_int = ni > p.o0 ? std::min(p.out_len, ni - p.o0) : 0;
    p.continues = !(s.eof && p.o_abs + p.out_len >= ready);
    if (s.run_cap && s.ends.size() > 1) {   // the current run is complete: the runs behind it that the block reaches
        uint64_t m = out_total(p.run_end - p.run_i, from, to) - p.o0;
        for (size_t k = 1; k < s.ends.size() && m < p.out_len; k++) {
            const uint64_t i = s.ends[k - 1], e = std::min(s.pushed, s.ends[k]);
            p.cuts.push_back(RunCut{m, i, e, std::min(p.out_len - m, out_interp(e - i, from, to))});
            m += out_total(e - i, from, to);
        }
    }
    return p;
}
// Mixer::add for a held source while the mixer has rendered T frames: it joins at the next frame (src/mixer.rs:175-183).
inline void start(Stream& s, uint64_t T) {
    if (s.held) s.held = false, s.mix_start = T;
}

// Skippable::skip / Player::skip_one / stop: the source's iterator returns None from now on.  The mixer's converter has pulled
// frames [0, fpos) of it (the right neighbour of the last rendered output included): those are its whole input now, the rest
// of the FIFO is forgotten.  A held source (or one that has rendered nothing yet: fpos = 0) ends empty.
inline void skip(Stream& s) {
    s.pushed = std::min(s.pushed, std::max(s.fpos, s.i0));
    s.eof = true;
    if (s.held) s.held = false, s.follows = -1, s.pushed = s.i0 = s.fpos = 0, s.out_done = 0, s.mix_start = 0;
    size_t keep = 0;           // runs none of whose frames is left never begin
    for (uint64_t i = s.run_i; keep < s.ends.size() && i < s.pushed; i = s.ends[keep++]) {}
    s.ends.resize(keep);
}

// After the block: advance the stream and tell how many FIFO frames (from the front) are dead.
inline uint64_t advance(Stream& s, const Part& p) {
    if (p.out_len) {   // the converter (and a filter in front of it) stands behind the right neighbour of the block's last output
        const RunCut* c = p.cuts.empty() ? nullptr : &p.cuts.back();   // ... in the run of that output: a new run pulls its first
        const uint64_t ia = ((c ? p.out_len - 1 - c->m : p.o0 + p.out_len - 1) * (uint64_t)s.from) / s.to;   // two frames at once
        s.fpos = std::min((c ? c->i : p.run_i) + ia + 2, c ? c->end : p.run_end);
    }
    s.out_done = p.out_len ? p.o_abs + p.out_len : s.out_done;
    settle(s);
    uint64_t left = std::min(s.run_i + ((s.out_done - s.run_o) * (uint64_t)s.from) / s.to, s.pushed);   // left frame of the next output
    if (s.front) left = std::min(left, s.fpos);   // more than two input frames per output: the filter still needs the ones between
    const uint64_t keep_from = left & ~3ull;                                        // FIFO front stays 16-byte aligned
    const uint64_t drop = keep_from > s.i0 ? keep_from - s.i0 : 0;
    s.i0 += drop;
    return drop;
}

}  // namespace session
