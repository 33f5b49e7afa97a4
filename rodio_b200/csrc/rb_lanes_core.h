// rb_lanes_core.h — the lane-per-stream fused kernel: resample (linear interpolation, from < to) -> [biquad] ->
// [one gain] -> mixer sum, for LARGE batches of mono or interleaved-stereo f32 streams that share one reduced rate ratio
// (template parameter C = channels of every stream and of the mixer; a stereo lane carries both channels of its stream:
// one index state, one 8-byte tap fetch per input frame, two filters).
//
// Why a second kernel next to k_fused_hot (rb_fused.cu).  The exact biquad is a serial chain per stream (bit
// parity with src/source/blt.rs:558-560 forbids re-association), so a stream can never run faster than one sample
// per ~13 cycles.  k_fused_hot answers that for a few thousand streams: one warp per SM runs nothing but the
// recurrences while the other warps do the time-parallel work for it -- the right shape at 28 streams per SM, but
// beyond that its throughput is flat (~33 issue slots per sample on three of the four SM sub-partitions, 25 % of
// the HBM roofline at 16 384 and 65 536 streams).  With hundreds of streams per SM the parallelism is across
// streams, so here EVERY lane owns one stream and walks it serially in time:
//   * no cross-lane traffic for the resampler or the filter: both taps, the numerator, the filter state live in
//     the lane's registers; 28.4 (mono) / 26.0 (stereo) issue slots per sample in the steady state by static count
//     (tools/sass_loop_count.py: index 6, interpolation with its exact division 6, feed-forward 3-5, recurrence 4,
//     gain 1, mixer sum 4, bookkeeping 3), spread over all four sub-partitions;
//   * a warp = 32 consecutive streams (insertion order) in lock step on the mixer timeline, TILE = 8 samples per
//     loop iteration (one basic block: the loads and index arithmetic of all 8 steps are hoisted above the
//     recurrence chain by the compiler);
//   * the mixer sum is a transposing warp-shuffle reduction (7 + 2 shuffles per 8 x 32 samples): lane 4p ends up
//     with the sum of timeline position p over the warp's 32 streams and stores it -- one partial row per warp,
//     added in warp order by k_sum_groups.  (Summation order differs from the reference's sequential order: the
//     tolerance class of the fused path, <= 1e-5 * peak, tested; RB_MIX_EXACT_ORDER keeps the bit-exact path.)
//   * inputs reach the lanes through a per-lane ring in shared memory filled by 16-byte cp.async (LDGSTS) in
//     64-byte chunks (16 mono / 8 stereo frames), two chunks ahead; the copies of a chunk are distributed so that 4 consecutive lanes fetch
//     64 contiguous bytes of one stream (coalesced sectors), whatever stream the copying lane itself owns.
//     Every input byte is read from HBM once; there are no intermediates in HBM.
// Streams that start late / end early / end in the "last frame raw" rule (sample_rate.rs:187-199) are handled by
// run management: the timeline is cut into FAST runs (every lane either fully interior or idle -- idle lanes walk
// a buffer of zeros) and single SLOW tiles (per-lane closed form with 64-bit index math, IEEE division, global
// loads), so the hot loop carries no per-lane activity predicates at all.
//
// Exact division.  The reference computes a + ((b-a)*num)/den with an IEEE division (src/math.rs:24-26).  The fast
// tile uses q0 = m*r, q = fma(fma(-q0, den, m), r, q0) with r = RN(1/den) -- correctly rounded whenever the
// residual is exact, i.e. for every m that is 0 or in [2^-100, 2^100) (verified against `/` on 136 M cases
// including every den <= 4000).  Instead of guarding every sample, streams are classified ONCE when their PCM is
// uploaded (k_classify_inputs: all non-zero |x| inside [2^-70, 2^60]); a stream outside that class never takes the
// fast path (its warp stays on slow tiles, which divide with __fdiv_rn).  Within the class (b-a)*num is 0 or at
// least 2^-94, so the quotient is exact.  The only visible difference is the sign of a zero quotient
// ((-0)/den = -0, here +0): it can flip the sign of an exactly-zero stream sample, never a non-zero one, and the
// mixer adds +0.0 last, as the reference's accumulator starts from it (src/mixer.rs:185-198).
//
// This header is compiled twice: by nvcc into k_fused_lanes (rb_lanes.cu) and by g++ into the CPU emulator of
// tests/emu/ (RB_SIMT_EMULATE), which runs the same warp program on 32 host threads against the oracle.
#pragma once
#include <cstdint>

#include "rb_simt.h"

namespace lanes {

constexpr int TILE = 8;                 // timeline SAMPLES per loop iteration (TILE / C frames)
#ifndef RB_LANES_STEREO_CHW
#define RB_LANES_STEREO_CHW 16
#endif
constexpr int CHUNK = 16;               // 32-bit words per ring chunk and lane (one cp.async group): 16 mono / 8 stereo frames
// Ring slots of the up-sampling / same-rate tiles.  4 (the measured geometry): chunk c-1 (draining), c, c+1 (in flight),
// c+2 (just issued) -- two chunks of look-ahead.  -DRB_LANES_UP_SLOTS=3 builds them with ONE chunk of look-ahead (a chunk is
// two tiles of work, several HBM latencies at the measured issue rate) and 68 instead of 84 words per lane: 24 instead of 20
// warps per SM.  Verified on the emulator, never timed: an A/B knob for the next device pass.  The DOWN tiles always have
// 4 slots and one chunk of look-ahead (see there).
#ifndef RB_LANES_UP_SLOTS
#define RB_LANES_UP_SLOTS 4
#endif
static_assert(RB_LANES_UP_SLOTS == 3 || RB_LANES_UP_SLOTS == 4, "3 (one chunk ahead) or 4 (two chunks ahead)");
constexpr int NSLOT_DOWN = 4;
constexpr uint32_t RUN_CAP = 1u << 30;  // frames
constexpr int MIN_RUN_TILES = 4;        // shortest fast run worth priming the ring for
// Per-lane ring geometry for C interleaved channels (C = 1 mono, 2 stereo); sizes in 32-bit words.
template <int C, int NSLOT = RB_LANES_UP_SLOTS>
struct Geo {
    static constexpr int TF = TILE / C;            // frames per tile
    // words per chunk: 64 bytes per lane for either layout.  (Stereo lanes had 16-frame chunks when the kernel first ran on
    // a device: 41 KB per CTA, 10 warps per SM.  Halved afterwards, not timed yet: -DRB_LANES_STEREO_CHW=32 rebuilds the
    // old geometry for an A/B run.)
    static constexpr int CHW = C == 2 ? RB_LANES_STEREO_CHW : CHUNK;
    static constexpr int CHF = CHW / C;            // frames per chunk
    static constexpr int RING = CHW * NSLOT;       // 64 words
    static constexpr int MIRROR = CHW;             // ring words [RING, RING + MIRROR) repeat [0, MIRROR): a tile never wraps
    static constexpr int RS = RING + MIRROR + 4;   // 84 words per lane; RS / 4 odd: 8 lanes hit 8 bank quads
    static constexpr int QPC = CHW / 4;            // 16-byte quads per chunk and stream
    static constexpr int RPI = 32 / QPC;           // streams served by one cp.async warp instruction
    static_assert(TILE % C == 0 && MIRROR >= TILE && (RS / 4) % 2 == 1 && 32 % QPC == 0 && CHW % (4 * C) == 0 && CHF >= 2 * (TILE / C), "ring geometry");
};
static_assert(RUN_CAP % TILE == 0, "run cap");
constexpr uint32_t ROW_UNSAFE = 1u;     // Row::flags: some sample outside the exact-reciprocal class
constexpr uint32_t ROW_CONTINUES = 2u;  // Row::flags: the stream goes on in the next block -- keep the filter state past `end`
constexpr uint32_t ROW_FORCE_SLOW = 4u; // Row::flags: set by the host (a gain in front of the conversion outside [2^-6, 2^6]): not on an
                                        // unguarded interpolating tile -- the host launches the GUARD twin for the class, or (DOWN) slow tiles

struct Row {                 // one stream (whole, or the part of it one block of a streaming session renders)
    const float* in;         // f32 frames (C interleaved channels), 16-byte aligned, readable up to a 16-byte tail pad
    uint64_t L;              // input frames at `in`
    uint64_t out_len;        // FRAMES on the (block's) mixer timeline
    uint64_t mix_start;      // timeline frame of the first of them
    uint64_t n_int;          // outputs [0, n_int) interpolate between two frames (left frame <= L-2)
    uint64_t o0;             // streaming: stream-absolute index of the first output of the block (0 for whole streams)
    uint64_t i0;             // streaming: stream-absolute index of the frame at in[0]; (o0 * from) / to >= i0
                             // (a session with restart schedules counts o0 and i0 from the first output and the first frame of the
                             // row's converter run: i0 is then taken modulo 2^64, in[0] may lie in front of the run)
    float* state;            // streaming: per channel {x[n-1], x[n-2], y[n-1], y[n-2]} (4*C floats) read at the start,
                             // written at the end; NULL: start from zeros, keep nothing
    float b0, b1, b2, a1, a2;
    float ffk;               // FF2 variant: b1 == ffk * b0 (ffk = +-2) and b2 == b0
    float post;              // the one gain behind the chain (NPOST == 1)
    float pre;               // PRE: the one gain in front of the conversion -- source.amplify(v) handed to the mixer, the
                             // usual rodio idiom -- applied to every input frame once, when it is fetched
    float mid;               // FRONT: the gain between the filter and the conversion (Player keeps its volume there)
    uint32_t flags;
    uint64_t f0;             // frames of in[] the converter had pulled when the block starts (0 for a whole stream): a FRONT filter
                             // has consumed them; the gain in front (PRE: pre, FRONT: mid) applies to frames >= f0 only ...
    float ga, gb;            // ... frame f0 - 2 was pulled with gain ga, frame f0 - 1 with gb (Player::set_volume between blocks:
                             // a frame keeps the factor it was multiplied with when Amplify::next pulled it)
};

// RESTART (streaming sessions): converter runs of the row end inside the block and the next ones begin -- rodio's
// UniformSourceIterator bootstraps a fresh SampleRateConverter there (src/source/uniform.rs:83-96), which interpolates inside
// itself only, emits its last frame raw and starts again at numerator 0 with two new frames.  The Row describes the run of the
// block's first output (L, n_int, o0, i0 up to its last frame); a row has any number of cuts, in timeline order, and from the
// block-local output m of each the lane walks that cut's run.  Filter state and gains pass through; a filter in FRONT consumes
// every input frame once, in order, across every cut.
struct Cut {
    uint64_t m;              // first output of the new run, relative to Row::mix_start (< Row::out_len, increasing along a row)
    uint64_t n_int;          // of the outputs [m, out_len) the first n_int interpolate
    uint64_t i0;             // Row::i0 of the new run, whose o0 is 0: its first frame is in[-i0] (modulo 2^64)
    uint64_t L;              // Row::L of the new run
};

// Optional per-group record (duo kernel, time-parallel plan): which partial row the group adds into, and from which timeline
// frame on its tiles are stored (what lies in front is the warm-up of a segment: computed, never stored).
struct GroupSpan {
    uint64_t store_lo;   // a multiple of TILE
    uint32_t slot, pad_;
};

struct Args {
    const Row* rows;
    uint32_t n_rows, n_groups;
    uint32_t from, to;       // reduced ratio, from < to <= 2^20
    uint32_t q8, r8;         // divmod((TILE / CO) * from, to): input frames a tile advances (CO = mixer channels)
    float den_f, rcp_den, from_f;
    uint32_t adv_q;          // DOWN: from / to, whole input frames per output (1 or 2) ...
    float rem_f;             // ... and from % to, what the numerator gains per output on top of them
    float neg1;              // -1.0f as a run-time value (keeps fma(p, -1, t) an FFMA: the chain stays on one pipe)
    uint64_t mix_len;        // mixer timeline, frames
    uint64_t pstride;        // floats per partial row: mix_len * CO rounded up to TILE
    float* partial;          // [n_groups][pstride], zero outside the span each group writes
    const float* zeros;      // CHUNK zeros, 16-byte aligned: the source of idle lanes
    const uint32_t* unsafe;  // optional [n_rows]: non-zero = as if ROW_UNSAFE were set (streaming: kept on the device)
    const GroupSpan* spans;  // optional [n_groups] (rb_duo_core.h)
    const Cut* cuts;         // RESTART: the cuts of row r are cuts[cut_first[r] .. cut_first[r + 1]) (compressed sparse rows)
    const uint32_t* cut_first;   // RESTART: [n_rows + 1]
};

// (t - a1*y1) - a2*y2, each product and each difference rounded once (src/source/blt.rs:558-560)
SIMT_FN float fb(float a1, float a2, float t, float y1, float y2, float neg1) {
    return simt::ffma(simt::fmul(a2, y2), neg1, simt::ffma(simt::fmul(a1, y1), neg1, t));
}

// Sum of v[u] over the 32 lanes for the 8 tile positions u; lane 4p receives position p.  Fixed tree.
SIMT_FN float reduce_tile(const float (&v)[TILE], uint32_t ln) {
    const bool b4 = ln & 16u, b3 = ln & 8u, b2 = ln & 4u;
    float w[4], z[2];
#pragma unroll
    for (int j = 0; j < 4; j++) w[j] = simt::fadd(b4 ? v[j + 4] : v[j], simt::shfl_xor(b4 ? v[j] : v[j + 4], 16));
#pragma unroll
    for (int j = 0; j < 2; j++) z[j] = simt::fadd(b3 ? w[j + 2] : w[j], simt::shfl_xor(b3 ? w[j] : w[j + 2], 8));
    float s = simt::fadd(b2 ? z[1] : z[0], simt::shfl_xor(b2 ? z[0] : z[1], 4));
    s = simt::fadd(s, simt::shfl_xor(s, 1));
    s = simt::fadd(s, simt::shfl_xor(s, 2));
    return simt::fadd(s, 0.0f);   // the reference's accumulator starts from +0.0: an all-(-0) column sums to +0
}

// PASS: the streams are at the mixer's rate already (reduced ratio 1:1): SampleRateConverter hands its input through
// untouched (src/conversions/sample_rate.rs:131-136), so the taps are used raw -- no interpolation, no division, and no
// input class to respect; everything else (ring, runs, "an output needs its successor or the end of the stream") is the
// same code with from = to = 1.
// CI / CO: channels of the streams of this launch / of the mixer.  CI == CO (mono into mono, stereo into stereo), or
// CI = 1, CO = 2: a mono source in a stereo mixer -- ChannelCountConverter repeats the sample on both channels
// (src/conversions/channels.rs:57-85) and the two filter channels see the same input, so the lane computes the frame once
// and emits it twice.
//
// FRONT: the biquad sits IN FRONT of the conversion -- `source.low_pass(f)` handed to Mixer::add or appended to a Player
// (src/player.rs:120-128: user source -> pausable -> amplify -> mixer's UniformSourceIterator).  The filter then runs once per
// INPUT frame, at the source's rate: frame * pre -> biquad -> * mid -> interpolation taps -> [* post].  The lane keeps the
// filter exactly one frame ahead of the interpolation (it has consumed frames [0, i + 2) when the output with left frame i
// is formed, or all L of them at the end), so the taps ARE y[n-2], y[n-1] (times `mid`) and no state is added.  Filter
// outputs cannot be classified in advance, so the division of the fast tile is guarded per sample (|m| inside
// [2^-100, 2^100) or zero: reciprocal step, else IEEE division).
//
// DOWN: sources above the mixer's rate, up to twice (48 kHz in a 44.1 kHz mixer, 96 kHz in a 48 kHz one) on fast tiles: every
// output moves on q = from / to whole frames (1 or 2) plus one more on a numerator carry, and reloads both taps from the
// ring; a tile consumes at most one chunk, so the refill logic is the one of the up-sampling tile.  Row::pre is always
// applied (no PRE twin).  Larger ratios stay on the slow tiles.  With FRONT the one or two frames an output moves on are
// one or two steps of the filter.
//
// RESTART: rows may change their converter run any number of times inside the block (Cut above).  A tile that holds a lane's cut
// is a slow tile -- the ending run's fast tiles stop where its interpolating outputs do -- whose closed form switches to the new
// run at the cut; a fast run between two cuts is primed from the new run's (o0 = 0, i0).
//
// GUARD (with PRE): some stream of the class has a gain in front outside [2^-6, 2^6] (a Player at -40 dB): its scaled taps may
// leave the range in which the reciprocal division is exact, so the tile checks every quotient like FRONT does and the
// stream stays on the fast tiles.  The host picks the variant per launch; rows and their order are the same, and so are the
// bits of every stream whose quotients were in range anyway.
template <int CI, int CO, bool HASB, bool FF2, int NPOST, bool PASS = false, bool PRE = false, bool FRONT = false, bool DOWN = false,
          bool GUARD = false, bool RESTART = false>
SIMT_FN void warp_main(const Args& a, uint32_t group, float* ring_warp) {
    static_assert(!GUARD || (PRE && !PASS), "GUARD: the guarded twin of the interpolating PRE variant");
    static_assert(!RESTART || !PASS, "RESTART: a same-rate conversion keeps nothing across a restart");
    static_assert(CI == CO || (CI == 1 && CO == 2), "channel layouts served");
    static_assert(!DOWN || (!PASS && !PRE), "DOWN: interpolating, the gain in front always applied");
    static_assert(!FRONT || (HASB && !FF2 && !PRE), "FRONT: plain coefficients, the gain in front is always applied");
    constexpr int NSLOT = DOWN ? NSLOT_DOWN : RB_LANES_UP_SLOTS;
    constexpr bool ONE_AHEAD = DOWN || RB_LANES_UP_SLOTS == 3;   // one chunk of look-ahead instead of two
    using G = Geo<CI, NSLOT>;
    constexpr int C = CI;               // taps, ring and filter state follow the source's channels
    constexpr int TF = TILE / CO;       // frames per tile: the mixer timeline has CO samples per frame
    constexpr int RS = G::RS, QPC = G::QPC, RPI = G::RPI, RING = G::RING, MIRROR = G::MIRROR, CHW = G::CHW, CHF = G::CHF;
    const uint32_t ln = simt::lane();
    const uint32_t r = group * 32u + ln;
    const bool has = r < a.n_rows;
    Row row;
    if (has) {
        row = a.rows[r];
    } else {
        row.in = a.zeros, row.L = 0, row.out_len = 0, row.mix_start = 0, row.n_int = 0, row.o0 = 0, row.i0 = 0, row.state = nullptr;
        row.b0 = row.b1 = row.b2 = row.a1 = row.a2 = row.ffk = row.post = row.pre = row.mid = row.ga = row.gb = 0.0f, row.flags = 0, row.f0 = 0;
    }
    uint64_t ms = row.mix_start, end = row.mix_start + row.out_len;   // frames; RESTART: of the run the lane is in
    uint64_t L = row.L, n_int = row.n_int;
    // Down-sampling classes (from > to: more than one input frame per output) are served by the slow tiles only -- exact,
    // general, not fast; the fast run below assumes at most one new frame per step.
    // (a same-rate stream never divides, a guarded tile checks every quotient: ROW_FORCE_SLOW means nothing to them)
    const bool safe = has && (a.from <= a.to || (DOWN && a.from <= 2 * a.to)) && (PASS || GUARD || !(row.flags & ROW_FORCE_SLOW)) &&
                      (PASS || FRONT || (!(row.flags & ROW_UNSAFE) && !(a.unsafe && a.unsafe[r])));
    bool stops = !(row.flags & ROW_CONTINUES);   // the stream ends inside this block (or is a whole stream)
    const bool live = has && row.out_len != 0;
    const uint64_t t_lo = simt::reduce_min64(live ? ms : ~0ull), t_hi = simt::reduce_max64(live ? end : 0ull);
    if (t_lo >= t_hi) return;
    const uint64_t t_end = (t_hi + TF - 1) / TF * TF;
    uint64_t t = t_lo / TF * TF;                        // timeline position in frames, a multiple of TF
    float* const ringl = ring_warp + ln * RS;
    float* const prow = a.partial + (uint64_t)group * a.pstride;
    const float den = a.den_f, rcp = a.rcp_den, from_f = a.from_f, neg1 = a.neg1;
    const float b0 = row.b0, b1 = row.b1, b2 = row.b2, a1 = row.a1, a2 = row.a2, ffk = row.ffk, post = row.post, gpre = row.pre, gmid = row.mid;
    const uint32_t from = a.from, to = a.to;
    uint64_t fpos = row.f0;   // FRONT: frames of in[] consumed by the filter
    // the gain in front for input frame k (relative to in[0]): frames the converter pulled in earlier blocks keep their factor
    const float gcur = FRONT ? gmid : gpre;
    const float rem_f = a.rem_f;
    const int adv_w0 = (int)a.adv_q * C, adv_w1 = adv_w0 + C;   // DOWN: ring words per output without / with a carry
    auto gain_of = [&](uint64_t k) { return k >= row.f0 ? gcur : (k + 1 == row.f0 ? row.gb : row.ga); };
    // canonical filter state per channel: x[n-1], x[n-2], y[n-1], y[n-2]
    float xh1[C], xh2[C], y1[C], y2[C];
#pragma unroll
    for (int c = 0; c < C; c++) {
        xh1[c] = xh2[c] = y1[c] = y2[c] = 0.f;
        if (HASB && row.state) xh1[c] = row.state[4 * c], xh2[c] = row.state[4 * c + 1], y1[c] = row.state[4 * c + 2], y2[c] = row.state[4 * c + 3];
    }
    // stream-absolute numerator of local output frame o is (o0 + o) * from; the input frame it falls on, relative to
    // in[0], is that / to - i0.  Both offsets are zero for whole streams.
    uint64_t o0 = row.o0, i0 = row.i0;
    // RESTART: the lane walks its current run up to timeline frame cut_t (the next cut) and moves to that cut's run when it gets
    // there; the last run ends with the row
    uint32_t ck = 0;
    uint64_t cut_t = ~0ull;
    if (RESTART && has) {
        ck = a.cut_first[r];
        if (ck < a.cut_first[r + 1]) cut_t = ms + a.cuts[ck].m, end = cut_t, stops = false;
    }
    auto restart_at = [&](uint64_t tt) {
        if (RESTART && tt >= cut_t) {   // (every run has an output: one cut per frame at most)
            const Cut cut = a.cuts[ck++];
            ms = cut_t, o0 = 0, i0 = cut.i0, L = cut.L, n_int = cut.n_int;
            if (ck < a.cut_first[r + 1]) {
                cut_t = row.mix_start + a.cuts[ck].m, end = cut_t;
            } else {
                cut_t = ~0ull, end = row.mix_start + row.out_len, stops = !(row.flags & ROW_CONTINUES);
            }
        }
    };
    const uint32_t cq = ln % QPC;                      // the quad of a chunk this lane copies ...
    const uint32_t cr = ln / QPC;                      // ... for stream cr + RPI * j of the warp
    // FRONT: one step of the filter on input frame `raw` (src/source/blt.rs:397-410 on src/source/amplify.rs:91-95)
    auto front_step = [&](const float (&raw)[C]) {
#pragma unroll
        for (int c = 0; c < C; c++) {
            const float x = simt::fmul(raw[c], gpre);
            const float ff = simt::fadd(simt::fadd(simt::fmul(b0, x), simt::fmul(b1, xh1[c])), simt::fmul(b2, xh2[c]));
            const float y = fb(a1, a2, ff, y1[c], y2[c], neg1);
            xh2[c] = xh1[c], xh1[c] = x, y2[c] = y1[c], y1[c] = y;
        }
    };
    // FRONT: let the filter consume in[fpos .. upto) from global memory (run starts, slow tiles)
    auto front_catch_up = [&](uint64_t upto) {
        while (fpos < upto) {
            float raw[C];
#pragma unroll
            for (int c = 0; c < C; c++) raw[c] = simt::ldg(row.in + fpos * C + c);
            front_step(raw);
            fpos++;
        }
    };

    while (t < t_end) {
        restart_at(t);
        // ---- how long does every lane stay "interior or idle" from t on? ----
        uint32_t d;
        if (!has || t >= end) {
            d = RUN_CAP;
            if (stops) {                                // a finished stream contributes nothing, its filter stops
#pragma unroll
                for (int c = 0; c < C; c++) xh1[c] = xh2[c] = y1[c] = y2[c] = 0.f;
            }
        } else if (t < ms) {
            const uint64_t g = (ms - t) / TF * TF;      // idle until the tile the stream starts in
            d = g > RUN_CAP ? RUN_CAP : (uint32_t)g;
        } else {
            const uint64_t o = t - ms;
            d = 0;
            // FRONT: the index step behind the last output of a run already feeds the NEXT frame to the filter, so that
            // output must be an interpolating one as well (its right neighbour exists): the run stops one output short
            const uint64_t n_fast = FRONT ? (n_int ? n_int - 1 : 0) : n_int;
            if (safe && o + TF <= n_fast) {
                const uint64_t g = (n_fast - o) / TF * TF;
                d = g > RUN_CAP ? RUN_CAP : (uint32_t)g;
            }
        }
        const uint64_t left = t_end - t;
        const uint32_t cap = left > RUN_CAP ? RUN_CAP : (uint32_t)left;
        const uint32_t run = simt::reduce_min(d < cap ? d : cap);   // frames, a multiple of TF

        if (run >= (uint32_t)(MIN_RUN_TILES * TF)) {
            // =================================== FAST RUN: `run` timeline frames ===================================
            const bool act = has && t >= ms && t < end;
            uint32_t num = 0, k0 = 0, maxq = QPC - 1;
            float g_tap0 = gcur, g_tap1 = gcur;          // the first two taps may have been pulled in an earlier block
            const float* src = a.zeros;
            if (act) {
                const uint64_t prod = (o0 + (t - ms)) * (uint64_t)from;
                const uint64_t ia = prod / to;
                num = (uint32_t)(prod - ia * to);
                const uint64_t i = ia - i0;
                const uint64_t ibase = i & ~3ull;       // a multiple of 4 frames: 16-byte aligned for either C
                k0 = (uint32_t)(i - ibase);
                src = row.in + ibase * C;
                const uint64_t mq = ((L * C - 1) >> 2) - ((ibase * C) >> 2);   // last quad (relative) that holds a frame
                maxq = mq > 0x7fffffffull ? 0x7fffffffu : (uint32_t)mq;
                if (FRONT) front_catch_up(i + 2);       // interior: i + 1 < L
                if (PRE || FRONT || DOWN) g_tap0 = gain_of(i), g_tap1 = gain_of(i + 1);
            }
            // the streams this lane copies for: source pointer and clamp of stream cr + RPI * j
            uint64_t sq[QPC];
            uint32_t mq[QPC];
#pragma unroll
            for (int j = 0; j < QPC; j++) {
                sq[j] = simt::shfl_idx64((uint64_t)(uintptr_t)src, cr + RPI * j);
                mq[j] = simt::shfl_idx(maxq, cr + RPI * j);
            }
            auto issue = [&](uint32_t c) {
                const uint32_t slot = c % NSLOT;
                const uint32_t want = c * QPC + cq;
#pragma unroll
                for (int j = 0; j < QPC; j++) {
                    const uint32_t off = want < mq[j] ? want : mq[j];
                    const float* s = (const float*)(uintptr_t)sq[j] + 4ull * off;
                    float* dst = ring_warp + (cr + RPI * j) * RS + slot * CHW + cq * 4;
                    simt::cp16(dst, s);
                    if (slot == 0 && (int)(cq * 4) < MIRROR) simt::cp16(dst + RING, s);
                }
                simt::cp_commit();
            };
            issue(0);
            issue(1);
            simt::cp_wait<1>();   // chunk 0 has landed
            simt::syncwarp();
            // DOWN looks one chunk ahead instead of two: a tile may consume a whole chunk, so the slowest lane can still be
            // reading chunk c_ready - 2 when chunk c_ready is waited for -- the new copy then goes into the slot of c_ready - 3
            if (!ONE_AHEAD) issue(2);
            uint32_t c_ready = 1;   // chunks [0, c_ready) are readable; c_ready and (two ahead) c_ready + 1 are in flight
            const simt::sptr ring_end = simt::sptr_of(ringl + RING);
            simt::sptr p = simt::sptr_of(ringl + k0 * C);
            float x0[C], x1[C];
#pragma unroll
            for (int c = 0; c < C; c++) {
                x0[c] = simt::lds(simt::sptr_add(p, c)), x1[c] = simt::lds(simt::sptr_add(p, C + c));
                if (PRE || (DOWN && !FRONT)) x0[c] = simt::fmul(x0[c], g_tap0), x1[c] = simt::fmul(x1[c], g_tap1);
                if (FRONT) x0[c] = simt::fmul(y2[c], g_tap0), x1[c] = simt::fmul(y1[c], g_tap1);   // the filter is one frame ahead
            }
            if (!DOWN || FRONT) p = simt::sptr_add(p, 2 * C);   // the next frame to fetch; DOWN (without FRONT) keeps the cursor on the left tap
            float nf = simt::u2f(num);
            // upper bound (in frames) of any lane's next ring frame after the coming tile: the lane with the largest phase
            uint32_t kb = 5, kbn = to - 1;
            float p1[C], p2[C];
#pragma unroll
            for (int c = 0; c < C; c++) {
                p1[c] = p2[c] = 0.f;
                if (HASB && FF2) p1[c] = simt::fmul(b0, xh1[c]), p2[c] = simt::fmul(b0, xh2[c]);
            }

            // One tile: ring bookkeeping, then TF frames per lane into v[].  The mixer sum of a tile (five dependent shuffle
            // levels, nothing in the tile left to overlap them) is issued one tile late, inside the next tile's basic block,
            // so that the scheduler can hide its latency behind that tile's loads and arithmetic.
            auto tile = [&](float (&v)[TILE]) {
                kb += a.q8, kbn += a.r8;
                if (kbn >= to) kbn -= to, kb += 1;
                if ((kb - 1) / CHF >= c_ready) {
                    if (ONE_AHEAD) {
                        simt::cp_wait<0>();      // chunk c_ready has landed
                        simt::syncwarp();        // ... for every lane, and nobody reads chunk c_ready + 1 - NSLOT any more
                        issue(c_ready + 1);      // into the slot of chunk c_ready + 1 - NSLOT (DOWN: c - 3, 3 slots: c - 2)
                    } else {
                        simt::cp_wait<1>();      // chunk c_ready has landed (c_ready + 1 may still be in flight)
                        simt::syncwarp();        // ... for every lane, and nobody reads chunk c_ready - 2 any more
                        issue(c_ready + 2);      // into the slot of chunk c_ready - 2
                    }
                    c_ready += 1;
                    simt::emu_count(2, 1);
                }
                if (simt::sptr_ge(p, ring_end)) p = simt::sptr_add(p, -RING);
#pragma unroll
                for (int f = 0; f < TF; f++) {
                    float x[C];
#pragma unroll
                    for (int c = 0; c < C; c++) {
                        if (PASS) {
                            x[c] = x0[c];
                        } else {
                            // src/math.rs:24-26: first + (second - first) * num / den, the division as an exact reciprocal step
                            const float m = simt::fmul(simt::fsub(x1[c], x0[c]), nf);
                            const float q0 = simt::fmul(m, rcp);
                            float q = simt::ffma(simt::ffma(-q0, den, m), rcp, q0);
                            if ((FRONT || GUARD) && !simt::in_exact_quotient_class(m)) q = simt::fdiv_cold(m, den), simt::emu_count(3, 1);   // filter tails: denormals
                            x[c] = simt::fadd(x0[c], q);
                        }
                    }
                    // next output frame: numerator += from (mod to); a carry moves one input frame on
                    if (DOWN && FRONT) {
                        const float nf2 = simt::fadd(nf, rem_f);
                        const bool carry = nf2 >= den;
                        nf = carry ? simt::fsub(nf2, den) : nf2;
                        // one or two frames per output = one or two filter steps: the first always, the second (a whole
                        // second frame per output at a ratio of two, else the carry) computed and committed by selects
                        const bool second = carry || a.adv_q == 2u;
#pragma unroll
                        for (int k = 0; k < 2; k++) {
                            const bool take = k == 0 || second;
#pragma unroll
                            for (int c = 0; c < C; c++) {
                                const float xin = simt::fmul(simt::lds(simt::sptr_add(p, c)), gpre);
                                const float ff = simt::fadd(simt::fadd(simt::fmul(b0, xin), simt::fmul(b1, xh1[c])), simt::fmul(b2, xh2[c]));
                                const float yn = fb(a1, a2, ff, y1[c], y2[c], neg1);
                                const float tap = simt::fmul(yn, gmid);
                                xh2[c] = take ? xh1[c] : xh2[c], xh1[c] = take ? xin : xh1[c];
                                y2[c] = take ? y1[c] : y2[c], y1[c] = take ? yn : y1[c];
                                x0[c] = take ? x1[c] : x0[c], x1[c] = take ? tap : x1[c];   // a tap keeps the factor it was pulled with
                            }
                            p = simt::sptr_add(p, take ? C : 0);
                            if (simt::sptr_ge(p, ring_end)) p = simt::sptr_add(p, -RING);
                        }
                    } else if (DOWN) {
                        const float nf2 = simt::fadd(nf, rem_f);
                        const bool carry = nf2 >= den;
                        nf = carry ? simt::fsub(nf2, den) : nf2;
                        p = simt::sptr_add(p, carry ? adv_w1 : adv_w0);
                        if (simt::sptr_ge(p, ring_end)) p = simt::sptr_add(p, -RING);
#pragma unroll
                        for (int c = 0; c < C; c++) {
                            x0[c] = simt::fmul(simt::lds(simt::sptr_add(p, c)), gpre);
                            x1[c] = simt::fmul(simt::lds(simt::sptr_add(p, C + c)), gpre);
                        }
                    } else if (FRONT) {
                        // The filter step sits on the carry of the index step (0.92 of the steps at 44.1 -> 48 kHz): computed
                        // on every step from the frame under the cursor and committed by selects -- no divergent branch; a
                        // frame that is not consumed (no carry) may not even have landed yet, its result is dropped.
                        const float nf2 = simt::fadd(nf, from_f);
                        const bool carry = nf2 >= den;
                        nf = carry ? simt::fsub(nf2, den) : nf2;
#pragma unroll
                        for (int c = 0; c < C; c++) {
                            const float xin = simt::fmul(simt::lds(simt::sptr_add(p, c)), gpre);
                            const float ff = simt::fadd(simt::fadd(simt::fmul(b0, xin), simt::fmul(b1, xh1[c])), simt::fmul(b2, xh2[c]));
                            const float yn = fb(a1, a2, ff, y1[c], y2[c], neg1);
                            const float tap = simt::fmul(yn, gmid);
                            xh2[c] = carry ? xh1[c] : xh2[c], xh1[c] = carry ? xin : xh1[c];
                            y2[c] = carry ? y1[c] : y2[c], y1[c] = carry ? yn : y1[c];
                            x0[c] = carry ? x1[c] : x0[c], x1[c] = carry ? tap : x1[c];
                        }
                        p = simt::sptr_add(p, carry ? C : 0);
                    } else {
                        simt::lerp_advance<C, PRE>(nf, x0, x1, p, from_f, den, gpre);
                    }
                    float val[C];
#pragma unroll
                    for (int c = 0; c < C; c++) {
                        float y = x[c];
                        if (HASB && !FRONT) {
                            float tt;
                            if (FF2) {
                                // b1*x1 = ffk*(b0*x1) and b2*x2 = b0*x2 exactly: one product per sample, same roundings
                                const float pz = simt::fmul(b0, x[c]);
                                tt = simt::fadd(simt::ffma(p1[c], ffk, pz), p2[c]);
                                p2[c] = p1[c], p1[c] = pz;
                            } else {
                                tt = simt::fadd(simt::fadd(simt::fmul(b0, x[c]), simt::fmul(b1, xh1[c])), simt::fmul(b2, xh2[c]));
                            }
                            xh2[c] = xh1[c], xh1[c] = x[c];
                            y = fb(a1, a2, tt, y1[c], y2[c], neg1);
                            y2[c] = y1[c], y1[c] = y;
                        }
                        val[c] = NPOST ? simt::fmul(y, post) : y;
                    }
#pragma unroll
                    for (int co = 0; co < CO; co++) v[f * CO + co] = val[co < C ? co : 0];
                }
            };
            float vp[TILE];
            tile(vp);
            for (uint32_t done = TF; done < run; done += TF) {
                float v[TILE];
                tile(v);
                const float s = reduce_tile(vp, ln);                              // the previous tile's sum
                if ((ln & 3u) == 0) prow[(t + done - TF) * CO + (ln >> 2)] = s;
#pragma unroll
                for (int u = 0; u < TILE; u++) vp[u] = v[u];
            }
            {
                const float s = reduce_tile(vp, ln);
                if ((ln & 3u) == 0) prow[(t + run - TF) * CO + (ln >> 2)] = s;
            }
            simt::cp_wait<0>();
            simt::syncwarp();
            simt::emu_count(0, run / TF);
            if (FRONT && act) {   // the taps are those of the output that follows the run: the filter is one frame ahead of them
                const uint64_t prod = (o0 + (t + run - ms)) * (uint64_t)from;
                fpos = prod / to - i0 + 2;
            }
            t += run;
        } else {
            // =================================== SLOW TILE: per-lane closed form ===================================
            float v[TILE];
#pragma unroll 1
            for (int f = 0; f < TF; f++) {
                const uint64_t tt = t + (uint64_t)f;
                restart_at(tt);
                const bool on = has && tt >= ms && tt < end;
                uint64_t i = 0;
                uint32_t num = 0;
                if (on) {
                    const uint64_t prod = (o0 + (tt - ms)) * (uint64_t)from;
                    const uint64_t ia = prod / to;
                    num = (uint32_t)(prod - ia * to);
                    i = ia - i0;
                } else if (has && tt >= end && stops) {
#pragma unroll
                    for (int c = 0; c < C; c++) xh1[c] = xh2[c] = y1[c] = y2[c] = 0.f;
                }
                if (FRONT && on) front_catch_up(i + 2 < L ? i + 2 : L);
                float val[C];
#pragma unroll
                for (int c = 0; c < C; c++) {
                    val[c] = 0.0f;
                    if (FRONT) {
                        if (on) {
                            // the filter has consumed frames [0, fpos): y1 = F[fpos - 1], y2 = F[fpos - 2]
                            const bool two = fpos == i + 2;
                            const float xa = simt::fmul(two ? y2[c] : y1[c], gain_of(i));
                            float x = xa;
                            if (!PASS && two) x = simt::fadd(xa, simt::fdiv(simt::fmul(simt::fsub(simt::fmul(y1[c], gain_of(i + 1)), xa), simt::u2f(num)), den));
                            val[c] = NPOST ? simt::fmul(x, post) : x;
                        }
                    } else if (on) {
                        float xa = simt::ldg(row.in + i * C + c);
                        if (PRE || DOWN) xa = simt::fmul(xa, gain_of(i));
                        float x = xa;
                        if (!PASS && i + 1 < L) {
                            float xb = simt::ldg(row.in + (i + 1) * C + c);
                            if (PRE || DOWN) xb = simt::fmul(xb, gain_of(i + 1));
                            x = simt::fadd(xa, simt::fdiv(simt::fmul(simt::fsub(xb, xa), simt::u2f(num)), den));
                        }
                        float y = x;
                        if (HASB) {
                            const float ff = simt::fadd(simt::fadd(simt::fmul(b0, x), simt::fmul(b1, xh1[c])), simt::fmul(b2, xh2[c]));
                            y = fb(a1, a2, ff, y1[c], y2[c], neg1);
                            xh2[c] = xh1[c], xh1[c] = x, y2[c] = y1[c], y1[c] = y;
                        }
                        val[c] = NPOST ? simt::fmul(y, post) : y;
                    }
                }
#pragma unroll
                for (int co = 0; co < CO; co++) v[f * CO + co] = val[co < C ? co : 0];
            }
            const float s = reduce_tile(v, ln);
            if ((ln & 3u) == 0) prow[t * CO + (ln >> 2)] = s;
            simt::emu_count(1, 1);
            t += TF;
        }
    }
    if (HASB && row.state) {
#pragma unroll
        for (int c = 0; c < C; c++) row.state[4 * c] = xh1[c], row.state[4 * c + 1] = xh2[c], row.state[4 * c + 2] = y1[c], row.state[4 * c + 3] = y2[c];
    }
}

}  // namespace lanes
