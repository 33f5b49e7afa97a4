// rb_api.cu — C ABI (include/rodio_b200.h), host-side planner and launch sequencing.
//
// The planner turns every rb_stream_desc (a SamplesBuffer + adapter chain handed to Mixer::add,
// reference src/mixer.rs:58-66) into a list of nodes with closed-form lengths, validates what the
// reference constructors would panic on, lays the streams out in HBM and records the launch list.
// Product code: there is no CPU compute path here — everything that touches samples is a kernel.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <numeric>
#include <string>
#include <vector>

#include "rb_internal.h"
#include "rb_fused.h"
#include "rb_lanes.h"
#include "rb_lanes_plan.h"
#include "rb_session_plan.h"
#include "rb_p2p.h"
#if defined(RB_SIMT_EMULATE)
#include "rb_master_host.h"   // the CPU build of the host code (tests/emu/): k_master's arithmetic in host form
#include "rb_session_host.h"  // ... and the sessions' FIFO scatter and slot sum
#endif

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static rb_status fail(rb_status s, const std::string& msg) {
    g_last_error = msg;
    return s;
}
#define RB_CUDA(expr)                                                                      \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            return fail(_e == cudaErrorMemoryAllocation ? RB_ERR_OUT_OF_MEMORY : RB_ERR_CUDA, \
                        std::string(#expr) + ": " + cudaGetErrorString(_e));               \
        }                                                                                  \
    } while (0)

extern "C" const char* rb_status_string(rb_status s) {
    switch (s) {
        case RB_OK: return "ok";
        case RB_ERR_INVALID_ARGUMENT: return "invalid argument";
        case RB_ERR_CUDA: return "CUDA error";
        case RB_ERR_OUT_OF_MEMORY: return "out of device memory";
        case RB_ERR_UNSUPPORTED: return "unsupported by the block path";
        case RB_ERR_UNALIGNED_FRAMES: return "input is not a whole number of frames";
        case RB_ERR_RATIO_OVERFLOW: return "reduced sample-rate ratio overflows rodio's u32 index math";
        case RB_ERR_NOT_SUPPORTED_SEEK: return "seek not supported";
        case RB_ERR_BUFFER_TOO_SMALL: return "output buffer too small";
        case RB_ERR_STATE: return "call order violated";
        default: return "unknown status";
    }
}
extern "C" const char* rb_last_error(void) { return g_last_error.c_str(); }
extern "C" uint32_t rb_abi_version(void) { return RB_ABI_VERSION; }

// ------------------------------------------------------------------------------------------------
// host restatements of rodio's pure helper functions (glibc libm == what rustc's std lowers to)
// ------------------------------------------------------------------------------------------------
namespace hostmath {
constexpr float PI_F = 3.14159265358979323846264338327950288f;
constexpr float LOG2_10_F = 3.32192809488736234787031942948939018f;
constexpr float LOG10_2_F = 0.301029995663981195213738894724493027f;

static float duration_secs_f32(uint64_t ns) {  // Duration::as_secs_f32
    uint64_t secs = ns / 1000000000ull;
    uint32_t nanos = (uint32_t)(ns % 1000000000ull);
    volatile float a = (float)secs;
    volatile float b = (float)nanos / 1000000000.0f;
    return a + b;
}
static float duration_to_coefficient(uint64_t ns, uint32_t rate) {  // src/math.rs:111-113
    volatile float d = duration_secs_f32(ns) * (float)rate;
    volatile float q = -1.0f / d;
    return expf(q);
}
struct Blt {
    float b0, b1, b2, a1, a2;
};
static Blt blt(bool high, uint32_t freq, float q, uint32_t fs) {  // src/source/blt.rs:502-544
    volatile float w0 = ((2.0f * PI_F) * (float)freq) / (float)fs;
    volatile float cw = cosf(w0);
    volatile float alpha = sinf(w0) / (2.0f * q);
    volatile float b0, b1, b2;
    if (!high) {
        b1 = 1.0f - cw;
        b0 = b1 / 2.0f;
        b2 = b0;
    } else {
        b0 = (1.0f + cw) / 2.0f;
        b1 = -1.0f - cw;
        b2 = b0;
    }
    volatile float a0 = 1.0f + alpha;
    volatile float a1 = -2.0f * cw;
    volatile float a2 = 1.0f - alpha;
    return {b0 / a0, b1 / a0, b2 / a0, a1 / a0, a2 / a0};
}
static float dist_sq(const float a[3], const float b[3]) {  // src/source/spatial.rs:19-24
    volatile float s = 0.0f;
    for (int i = 0; i < 3; i++) {
        volatile float d = a[i] - b[i];
        volatile float dd = d * d;
        s = s + dd;
    }
    return s;
}
static void spatial_volumes(const float e[3], const float l[3], const float r[3], float out[2]) {  // spatial.rs:48-69
    volatile float lds = dist_sq(l, e), rds = dist_sq(r, e);
    volatile float max_diff = sqrtf(dist_sq(l, r));
    volatile float ld = sqrtf(lds), rd = sqrtf(rds);
    volatile float t1 = (ld - rd) / max_diff;
    volatile float t2 = (t1 + 1.0f) / 4.0f;
    volatile float ldm = fminf(t2 + 0.5f, 1.0f);
    volatile float u1 = (rd - ld) / max_diff;
    volatile float u2 = (u1 + 1.0f) / 4.0f;
    volatile float rdm = fminf(u2 + 0.5f, 1.0f);
    volatile float ldist = fminf(1.0f / lds, 1.0f);
    volatile float rdist = fminf(1.0f / rds, 1.0f);
    out[0] = ldm * ldist;
    out[1] = rdm * rdist;
}
static uint32_t f32_as_u32(float v) {  // Rust `as u32`
    if (!(v == v) || v <= 0.0f) return 0;
    if (v >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)v;
}
}  // namespace hostmath

// RB_FX_LIMIT -> the limiter's coefficients at `rate` (limit.rs:94-130, :877)
static rb_lim_params limit_params(const rb_effect& e, uint32_t rate) {
    rb_lim_params l;
    l.threshold = e.f32[0], l.knee = e.f32[1];
    volatile float k8 = 8.0f * e.f32[1];
    l.inv_knee_8 = 1.0f / k8;
    l.attack = hostmath::duration_to_coefficient(e.ns[0], rate);
    l.release = hostmath::duration_to_coefficient(e.ns[1], rate);
    return l;
}

// Adapters on the MixerSource: [AMPLIFY] [LIMIT] [AMPLIFY], each optional, at least one; the limiter is built for the mixer's
// rate (its channel count and rate never change: MixerSource::current_span_len() is None, mixer.rs:89-91).
static rb_status parse_master(const rb_effect* fx, uint32_t n, uint32_t mixer_rate, rb_master_params* out) {
    if (n && !fx) return fail(RB_ERR_INVALID_ARGUMENT, "effects is NULL");
    rb_master_params p{};
    p.pre = p.post = 1.0f;
    uint32_t i = 0;
    if (i < n && fx[i].kind == RB_FX_AMPLIFY) p.has_pre = 1, p.pre = fx[i++].f32[0];
    if (i < n && fx[i].kind == RB_FX_LIMIT) p.has_lim = 1, p.lim = limit_params(fx[i++], mixer_rate);
    if (i < n && fx[i].kind == RB_FX_AMPLIFY) p.has_post = 1, p.post = fx[i++].f32[0];
    if (i != n) return fail(RB_ERR_UNSUPPORTED, "master chain: [AMPLIFY] [LIMIT] [AMPLIFY] on the MixerSource, nothing else");
    *out = p;
    return RB_OK;
}

// ---- WAV ingest: where the samples are and what they are (src/decoder/wav.rs:119-151 names the formats rodio reads) ----
extern "C" rb_status rb_wav_parse(const void* image, uint64_t n, rb_wav_info* out) {
    if (!image || !out) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    const uint8_t* p = (const uint8_t*)image;
    auto u16 = [&](uint64_t o) { return (uint32_t)p[o] | ((uint32_t)p[o + 1] << 8); };
    auto u32 = [&](uint64_t o) { return u16(o) | (u16(o + 2) << 16); };
    if (n < 12 || memcmp(p, "RIFF", 4) != 0 || memcmp(p + 8, "WAVE", 4) != 0) return fail(RB_ERR_INVALID_ARGUMENT, "not a RIFF/WAVE image");
    memset(out, 0, sizeof(*out));
    bool have_fmt = false, have_data = false;
    uint32_t tag = 0;
    for (uint64_t o = 12; o + 8 <= n;) {
        const uint64_t len = u32(o + 4), body = o + 8;
        if (memcmp(p + o, "fmt ", 4) == 0) {
            if (len < 16 || body + 16 > n) return fail(RB_ERR_INVALID_ARGUMENT, "WAV: truncated fmt chunk");
            tag = u16(body), out->channels = (uint16_t)u16(body + 2), out->sample_rate = u32(body + 4), out->bits_per_sample = (uint16_t)u16(body + 14);
            if (tag == 0xFFFEu) {   // WAVE_FORMAT_EXTENSIBLE: the real tag is the first two bytes of the sub-format GUID
                if (len < 40 || body + 40 > n) return fail(RB_ERR_INVALID_ARGUMENT, "WAV: truncated extensible fmt chunk");
                tag = u16(body + 24);
            }
            have_fmt = true;
        } else if (memcmp(p + o, "data", 4) == 0) {
            out->data_offset = body;
            out->data_bytes = body + len <= n ? len : n - body;
            have_data = true;
            break;
        }
        o = body + len + (len & 1);   // chunks are word aligned
    }
    if (!have_fmt || !have_data) return fail(RB_ERR_INVALID_ARGUMENT, "WAV: no fmt or no data chunk");
    if (out->channels == 0 || out->sample_rate == 0) return fail(RB_ERR_INVALID_ARGUMENT, "WAV: zero channels or sample rate");
    const uint32_t bits = out->bits_per_sample;
    if (tag == 3u && bits == 32) out->format = RB_FMT_F32;
    else if (tag == 1u && bits == 8) out->format = RB_FMT_U8;
    else if (tag == 1u && bits == 16) out->format = RB_FMT_I16;
    else if (tag == 1u && bits == 24) out->format = RB_FMT_I24_IN_I32, out->packed24 = 1;
    else if (tag == 1u && bits == 32) out->format = RB_FMT_I32;
    else return fail(RB_ERR_UNSUPPORTED, "WAV: a sample format rodio's decoder does not read (tag " + std::to_string(tag) + ", " + std::to_string(bits) + " bits)");
    const uint64_t bytes_per = bits / 8;
    out->n_samples = out->data_bytes / bytes_per;
    out->n_samples -= out->n_samples % out->channels;    // whole frames
    out->data_bytes = out->n_samples * bytes_per;
    return RB_OK;
}
extern "C" void rb_wav_unpack24(const void* packed, uint64_t n_samples, int32_t* out) {
    const uint8_t* p = (const uint8_t*)packed;
    for (uint64_t i = 0; i < n_samples; i++) {
        const uint32_t v = (uint32_t)p[3 * i] | ((uint32_t)p[3 * i + 1] << 8) | ((uint32_t)p[3 * i + 2] << 16);
        out[i] = (int32_t)(v << 8) >> 8;   // sign-extend bit 23
    }
}

extern "C" uint32_t rb_speed_sample_rate(uint32_t input_rate, float factor) {  // src/source/speed.rs:130-133
    volatile float r = (float)input_rate * factor;
    return hostmath::f32_as_u32(fmaxf(r, 1.0f));
}
extern "C" uint64_t rb_delay_samples(uint64_t ns, uint32_t rate, uint16_t ch) {  // src/source/delay.rs:8-16
    unsigned __int128 s = (unsigned __int128)ns * ch * rate / 1000000000ull;
    return (uint64_t)s;
}
extern "C" float rb_db_to_linear(float d) {
    volatile float t = d * 0.05f;
    volatile float u = t * hostmath::LOG2_10_F;
    return powf(2.0f, u);
}
extern "C" float rb_linear_to_db(float l) {
    volatile float t = log2f(l) * hostmath::LOG10_2_F;
    return t * 20.0f;
}
extern "C" void rb_spatial_volumes(const float e[3], const float l[3], const float r[3], float out[2]) {
    hostmath::spatial_volumes(e, l, r, out);
}

// Output frames of SampleRateConverter on L input frames with reduced ratio from:to
// (closed form of src/conversions/sample_rate.rs:131-201; derivation in DESIGN.md).
static uint64_t src_out_frames(uint64_t L, uint32_t from, uint32_t to) {
    if (from == to) return L;
    if (L == 0) return 0;
    unsigned __int128 a = (unsigned __int128)(L - 1) * to;
    unsigned __int128 nstar = (a + from - 1) / from;                 // first n with floor(n*from/to) >= L-1
    bool raw = nstar * from < (unsigned __int128)L * to;             // ... and it is exactly L-1
    return (uint64_t)nstar + (raw ? 1 : 0);
}

static size_t fmt_size(uint32_t fmt) {
    switch (fmt) {
        case RB_FMT_F32: case RB_FMT_I32: case RB_FMT_I24_IN_I32: return 4;
        case RB_FMT_I16: case RB_FMT_U16: return 2;
        default: return 1;
    }
}

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
struct rb_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    int sm_count = 0;
};

extern "C" rb_status rb_context_create(int device, rb_context** out) {
    if (!out) return fail(RB_ERR_INVALID_ARGUMENT, "out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(RB_ERR_CUDA, std::string("no usable CUDA device (there is no CPU fallback): ") +
                                     cudaGetErrorString(e));
    if (device < 0 || device >= n) return fail(RB_ERR_INVALID_ARGUMENT, "device ordinal out of range");
    RB_CUDA(cudaSetDevice(device));
    auto ctx = std::make_unique<rb_context>();
    ctx->device = device;
    RB_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    RB_CUDA(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device));
    *out = ctx.release();
    return RB_OK;
}
extern "C" rb_status rb_context_destroy(rb_context* ctx) {
    if (!ctx) return RB_OK;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return RB_OK;
}
extern "C" rb_status rb_context_sync(rb_context* ctx) {
    if (!ctx) return fail(RB_ERR_INVALID_ARGUMENT, "ctx is NULL");
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    return RB_OK;
}
extern "C" rb_status rb_context_stream(rb_context* ctx, void** out) {
    if (!ctx || !out) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = (void*)ctx->stream;
    return RB_OK;
}
extern "C" rb_status rb_context_sm_count(rb_context* ctx, int* out) {
    if (!ctx || !out) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = ctx->sm_count;
    return RB_OK;
}

// ------------------------------------------------------------------------------------------------
// planner
// ------------------------------------------------------------------------------------------------
struct PlanNode {
    rb_node_dev d{};       // src/dst filled at layout time
    uint32_t rate_out = 0;
    uint32_t span_out = 0;
    uint32_t level = 0;    // launch level: one more than the node in front, for a MIX also behind the second input's last node
    int64_t other = -1;    // RB_N_MIX2: the stream whose final samples are the second input
    // from_iter: an adapter that starts from scratch at a span boundary (AGC, limiter) is launched as one node per run of samples
    struct Split {
        uint64_t off, n;   // samples
        rb_node_dev d;     // the run's parameters (kind, coefficients, channels); src / dst / aux are filled at layout time
    };
    std::vector<Split> splits;
};
struct PlanStream {
    rb_stream_desc desc{};
    std::vector<rb_effect> fx;
    std::vector<PlanNode> nodes;
    uint64_t out_len = 0;      // samples reaching the mixer
    uint64_t mix_start = 0;
    uint64_t chain_len = 0;    // samples of the chain itself (before the mixer's UniformSourceIterator)
    uint32_t chain_channels = 0, chain_rate = 0;
    // layout
    size_t in_off = 0;         // byte offset in the input arena
    size_t buf_off = 0;        // float offset in each ping-pong arena
    uint64_t buf_cap = 0;      // floats
    const float* final_ptr = nullptr;
    // second input of another stream's RB_FX_MIX (mix_start == RB_MIX_START_CONSUMED): never added to the mixer
    bool consumed = false, planned = false, planning = false;
    int64_t consumer = -1;
    uint32_t end_span = 0;     // what the end of the chain reports / leaves for the UniformSourceIterator that wraps it
    uint64_t end_tail_pad = 0;
    int64_t end_cv_last = -1;
    // source::from_iter (RB_FX_APPEND): this stream is the head of a sequence of buffers with their own formats, or one of the
    // buffers appended to a head.  The samples of the sequence are contiguous in the input arena (head first).
    int64_t appended_to = -1;
    std::vector<size_t> appended;          // head: the descriptors that follow it, in order
    uint64_t seq_samples = 0;              // head: samples of the whole sequence
    struct Run {                           // one UniformSourceIterator bootstrap of the mixer's conversion (uniform.rs:50-68)
        PlanNode nd;
        uint64_t in_off, out_off;          // samples into the sequence / into the converted stream
    };
    std::vector<Run> runs;
    uint32_t run_level = 0;
};

static rb_uniform_seg uniform_seg(uint64_t in_samples, uint32_t c_in, uint32_t c_out, uint32_t from, uint32_t to) {
    rb_uniform_seg g{};
    g.L = in_samples / c_in;
    g.p = (uint32_t)(in_samples % c_in);
    if (from == to) {
        g.full_out_frames = g.L;
        g.flat_total = in_samples;
    } else if (g.p == 0) {
        g.full_out_frames = src_out_frames(g.L, from, to);
        g.flat_total = g.full_out_frames * c_in;
    } else {
        // channels < p own L+1 frames; the others own L and never get their raw last frame
        uint64_t n_a = 0;
        if (g.L >= 1) {
            unsigned __int128 a = (unsigned __int128)(g.L - 1) * to;
            n_a = (uint64_t)((a + from - 1) / from);
        }
        g.full_out_frames = n_a;
        g.flat_total = n_a * c_in + (src_out_frames(g.L + 1, from, to) - n_a) * g.p;
    }
    // ChannelCountConverter over the flat sequence: whole groups of c_in, then a trailing group that
    // stops at the first missing input sample.
    uint64_t groups = g.flat_total / c_in, k = g.flat_total % c_in;
    g.out_samples = groups * c_out + std::min<uint64_t>(k, c_out);
    return g;
}

// `cv_last_frame_start` >= 0: the input is a ChannelVolume/Spatial over a SamplesBuffer whose last output
// frame starts there.  ChannelVolume forwards the *buffer's* span report (channel_volume.rs:106-108), and an
// exhausted SamplesBuffer reports Some(0) (buffer.rs:76-82): a re-bootstrap that lands inside the last
// frame therefore gets an empty Take and the rest of that frame is never pulled.
static rb_status plan_uniform(PlanNode& nd, uint64_t n_in, uint32_t c_in, uint32_t rate_in, uint32_t span_in,
                              uint32_t c_out, uint32_t rate_out, int64_t cv_last_frame_start = -1) {
    if (c_out == 0 || rate_out == 0) return fail(RB_ERR_INVALID_ARGUMENT, "uniform: zero channels or rate");
    if (c_out > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "uniform: more than 12 channels");
    uint32_t g = std::gcd(rate_in, rate_out);
    uint32_t from = rate_in / g, to = rate_out / g;
    if (from != to && (uint64_t)from * to >= (1ull << 32))
        return fail(RB_ERR_RATIO_OVERFLOW, "reduced from*to >= 2^32 (sample_rate.rs:45-47)");
    rb_uniform_params u{};
    u.from = from, u.to = to;
    uint64_t chunk = 0;
    if (span_in != 0) {
        chunk = std::min(span_in, RB_UNIFORM_SPAN_CAP);   // uniform.rs:56
        if (chunk >= n_in) chunk = 0;                      // a single chunk
    }
    if (chunk && cv_last_frame_start >= 0) {
        uint64_t B = ((uint64_t)cv_last_frame_start / chunk + 1) * chunk;   // first re-bootstrap inside the last frame
        if (B < n_in) n_in = B;
    }
    if (chunk) {
        u.chunk_samples = chunk;
        u.n_full_chunks = n_in / chunk;
        u.full = uniform_seg(chunk, c_in, c_out, from, to);
        u.tail = uniform_seg(n_in % chunk, c_in, c_out, from, to);
    } else {
        u.tail = uniform_seg(n_in, c_in, c_out, from, to);
    }
    nd.d.kind = RB_N_UNIFORM;
    nd.d.c_in = c_in, nd.d.c_out = c_out;
    nd.d.n_in = n_in, nd.d.n_out = u.n_full_chunks * u.full.out_samples + u.tail.out_samples;
    nd.d.p.uni = u;
    nd.rate_out = rate_out;
    nd.span_out = 0;   // UniformSourceIterator::current_span_len() == None (uniform.rs:108-110)
    return RB_OK;
}

// ---- source::from_iter of buffers with different formats (RB_FX_APPEND) ---------------------------------------------------------
// The host walks the CONTROL FLOW of rodio's adapters over such a source -- which span length and format FromIter reports when
// an adapter asks (from_iter.rs:83-109: the current buffer's while it is not exhausted, None once it is; the next buffer is only
// fetched inside next()) -- and turns it into closed forms: coefficient changes for a filter, converter runs for the mixer.
struct SeqSeg {
    uint64_t n;          // samples
    uint32_t c, r;       // channels, sample rate (after any Speed)
    bool spans;          // SamplesBuffer: Some(len) until exhausted; TestSource-like: None
};
// SpanTracker::advance (span.rs:66-101) over what FromIter reports, as events: `at` = flat index of the first sample that sees the
// new parameters, `seg` = the buffer whose format they are.  The same list serves a tracker that runs behind the sample (filters,
// limiter: blt.rs:122, limit.rs:651) and one that runs in front of the next pull (AGC, agc.rs:525): both notice the change between
// the first and the second sample of the new buffer -- FromIter fetches a buffer inside next(), so the first sample is out before
// anybody sees the new format.
struct SpanEvent {
    uint64_t at;
    size_t seg;
};
static std::vector<SpanEvent> span_events(const std::vector<SeqSeg>& segs) {
    std::vector<SpanEvent> ev;
    uint64_t counted = 0, g0 = 0, cached = 0;
    bool counting = false;       // cached_span_len is Some
    uint32_t last_c = segs[0].c, last_r = segs[0].r;
    for (size_t k = 0; k < segs.size(); k++) {
        const SeqSeg& g = segs[k];
        if (g.n == 0) continue;
        // behind sample j of this buffer the span is Some(g.n) for j < g.n - 1 and None behind the last one (exhausted); only the
        // first of them can see a boundary: the counter restarts there or the parameters are equal from then on
        if (g.spans && g.n >= 2) {
            const uint64_t cnt = counted + 1;
            const bool known = counting ? cnt >= cached : true;     // None: compare on every sample
            bool changed = false, boundary = false;
            if (known) {
                changed = g.c != last_c || g.r != last_r;
                last_c = g.c, last_r = g.r;
                boundary = counting ? true : changed;
            }
            if (boundary) counting = true, cached = g.n, counted = 0;
            else counted = cnt;
            if (boundary && changed) ev.push_back({g0 + 1, k});
            counted += g.n - 1;      // the other samples of the buffer: no boundary (counter below the span, or nothing changed)
        } else {
            counted += g.n;          // None behind every sample: the counter runs, nothing is compared
        }
        g0 += g.n;
    }
    return ev;
}
static rb_status plan_varying(PlanStream& ps, std::vector<SeqSeg> segs, size_t fx_from, uint16_t mixer_ch, uint32_t mixer_rate) {
    uint64_t n = 0;
    for (const SeqSeg& g : segs) n += g.n;
    const uint32_t c0 = segs[0].c;
    for (size_t fi = fx_from; fi < ps.fx.size(); fi++) {
        const rb_effect& e = ps.fx[fi];
        PlanNode nd;
        nd.d.c_in = nd.d.c_out = c0, nd.d.n_in = nd.d.n_out = n;   // c_in: the state layout a filter chose at construction (blt.rs:247-283)
        nd.rate_out = segs[0].r, nd.span_out = 0;
        switch (e.kind) {
            case RB_FX_AMPLIFY:
                nd.d.kind = RB_N_AMPLIFY, nd.d.p.amp.factor = e.f32[0];
                break;
            case RB_FX_SPEED:   // Speed::sample_rate() scales whatever its input reports at that moment (speed.rs:130-133)
                for (SeqSeg& g : segs) g.r = rb_speed_sample_rate(g.r, e.f32[0]);
                continue;
            case RB_FX_LOW_PASS:
            case RB_FX_HIGH_PASS: {
                const bool high = e.kind == RB_FX_HIGH_PASS;
                hostmath::Blt k = hostmath::blt(high, e.u32[0], e.f32[0], segs[0].r);
                nd.d.kind = RB_N_BIQUAD;
                nd.d.p.blt.b0 = k.b0, nd.d.p.blt.b1 = k.b1, nd.d.p.blt.b2 = k.b2, nd.d.p.blt.a1 = k.a1, nd.d.p.blt.a2 = k.a2;
                uint32_t n_sw = 0;
                for (const SpanEvent& ev : span_events(segs)) {
                    if (n_sw >= RB_MAX_BLT_SWITCH) return fail(RB_ERR_UNSUPPORTED, "from_iter: more format changes than a filter follows");
                    hostmath::Blt kk = hostmath::blt(high, e.u32[0], e.f32[0], segs[ev.seg].r);
                    nd.d.p.blt.sw_at[n_sw] = ev.at;      // the sample that crossed the boundary still had the old coefficients
                    float* d = nd.d.p.blt.sw_k[n_sw];
                    d[0] = kk.b0, d[1] = kk.b1, d[2] = kk.b2, d[3] = kk.a1, d[4] = kk.a2;
                    n_sw++;
                }
                nd.d.p.blt.n_sw = n_sw;
                break;
            }
            case RB_FX_AGC: {
                // agc.rs:524-548: the tracker in FRONT of every pull; a changed format recomputes the coefficients and starts the RMS
                // window, the peak follower and the gain from scratch -- from the second sample of the new span on (the first one is
                // pulled before FromIter reports the new buffer).  Every stretch between two such points is an AGC of its own.
                const float mg = e.f32[1];
                if (!(mg >= 0.1f)) return fail(RB_ERR_INVALID_ARGUMENT, "agc: clamp(0.1, absolute_max_gain) would panic");
                const uint64_t ten = 10ull * 1000000000ull;
                auto params = [&](uint32_t rate) {
                    rb_node_dev d{};
                    d.kind = RB_N_AGC, d.c_in = d.c_out = c0;
                    d.p.agc.target = e.f32[0], d.p.agc.max_gain = mg, d.p.agc.floor = e.f32[2];
                    d.p.agc.attack = hostmath::duration_to_coefficient(std::min(e.ns[0], ten), rate);
                    d.p.agc.release = hostmath::duration_to_coefficient(std::min(e.ns[1], ten), rate);
                    return d;
                };
                nd.d = params(segs[0].r);
                nd.d.n_in = nd.d.n_out = n;
                uint64_t from = 0;
                rb_node_dev cur = nd.d;
                for (const SpanEvent& ev : span_events(segs)) {
                    if (ev.at >= n) break;
                    nd.splits.push_back({from, ev.at - from, cur});
                    from = ev.at, cur = params(segs[ev.seg].r);
                }
                if (!nd.splits.empty()) nd.splits.push_back({from, n - from, cur});
                break;
            }
            case RB_FX_LIMIT: {
                // limit.rs:651-697: the tracker BEHIND the sample; another channel count rebuilds the per-channel state, the
                // coefficients (of the rate at construction) stay
                rb_node_dev base{};
                base.kind = RB_N_LIMIT, base.c_in = base.c_out = c0;
                base.p.lim = limit_params(e, segs[0].r);
                nd.d = base;
                nd.d.n_in = nd.d.n_out = n;
                uint64_t from = 0;
                rb_node_dev cur = base;
                for (const SpanEvent& ev : span_events(segs)) {
                    if (ev.at >= n || segs[ev.seg].c == cur.c_in) continue;
                    nd.splits.push_back({from, ev.at - from, cur});
                    from = ev.at, cur.c_in = cur.c_out = segs[ev.seg].c;
                }
                if (!nd.splits.empty()) nd.splits.push_back({from, n - from, cur});
                break;
            }
            case RB_FX_APPEND: return fail(RB_ERR_INVALID_ARGUMENT, "from_iter: APPEND only at the front of the chain");
            default: return fail(RB_ERR_UNSUPPORTED, "from_iter: amplify, speed, low_pass, high_pass, automatic_gain_control and limit follow a source whose format changes");
        }
        nd.level = ps.nodes.empty() ? 0u : ps.nodes.back().level + 1u;
        ps.nodes.push_back(nd);
    }
    ps.chain_len = n, ps.chain_channels = segs[0].c, ps.chain_rate = segs[0].r;
    ps.planning = false, ps.planned = true;
    if (ps.consumed) return fail(RB_ERR_UNSUPPORTED, "from_iter: such a source cannot be the second input of a mix");
    // Mixer::add: UniformSourceIterator::new(source, mixer_ch, mixer_rate) -- one converter run per bootstrap (uniform.rs:50-68,:83-96)
    uint64_t pos = 0, out = 0;
    size_t cur = 0;              // FromIter's current buffer (only next() moves on)
    uint64_t pulled = 0;         // samples pulled from it
    while (true) {
        const SeqSeg& g = segs[cur];
        const bool exhausted = pulled >= g.n;
        const bool some = g.spans && !exhausted;
        const uint64_t take = some ? std::min<uint64_t>(g.n, RB_UNIFORM_SPAN_CAP) : ~0ull;
        const uint64_t m = std::min<uint64_t>(take, n - pos);
        if (m == 0) break;
        PlanStream::Run run;
        rb_status s = plan_uniform(run.nd, m, g.c, g.r, 0, mixer_ch, mixer_rate, -1);
        if (s != RB_OK) return s;
        if (run.nd.d.n_out == 0) break;      // the bootstrap's first next() is None: the UniformSourceIterator ends here
        run.in_off = pos, run.out_off = out;
        ps.runs.push_back(run);
        pos += m, out += run.nd.d.n_out;
        uint64_t left = m;                   // FromIter::next moved through the buffers
        while (left) {
            const uint64_t here = std::min<uint64_t>(left, segs[cur].n - pulled);
            pulled += here, left -= here;
            if (left) cur++, pulled = 0;
            while (left && segs[cur].n == 0) cur++;
        }
    }
    ps.run_level = ps.nodes.empty() ? 0u : ps.nodes.back().level + 1u;
    ps.out_len = out;
    ps.mix_start = (ps.desc.mix_start + mixer_ch - 1) / mixer_ch * mixer_ch;
    return RB_OK;
}

// The closed-form adapters DISTORTION, LINEAR_RAMP and TAKE_DURATION on a stream of `c` channels whose input reports `rate`:
// kind and parameters of the node.  A take's count is the samples it emits before `remaining < dps` (0 when dps is 0); the batch
// planner bounds it by the input's length, the sessions' push programs by the frames pushed.
static rb_status plan_pointwise(const rb_effect& e, uint32_t rate, uint32_t c, rb_node_dev& d) {
    switch (e.kind) {
        case RB_FX_DISTORTION:
            if (!(e.f32[1] >= 0.0f)) return fail(RB_ERR_INVALID_ARGUMENT, "distortion: clamp(-t, t) panics for t < 0 or NaN");
            d.kind = RB_N_DISTORT, d.p.dist.gain = e.f32[0], d.p.dist.threshold = e.f32[1];
            return RB_OK;
        case RB_FX_LINEAR_RAMP:
            if (e.ns[0] == 0) return fail(RB_ERR_INVALID_ARGUMENT, "linear_gain_ramp: duration must be greater than zero");
            d.kind = RB_N_RAMP;
            d.p.ramp.total_ns = e.ns[0], d.p.ramp.dt_ns = 1000000000ull / rate;   // linear_ramp.rs:97-99
            d.p.ramp.start = e.f32[0], d.p.ramp.end = e.f32[1], d.p.ramp.clamp_end = e.u32[0] ? 1u : 0u;
            return RB_OK;
        default: {   // RB_FX_TAKE_DURATION
            const uint64_t dps = 1000000000ull / ((uint64_t)rate * c);                   // take.rs:65-69
            d.kind = RB_N_TAKE;
            d.p.take.total_ns = e.ns[0], d.p.take.dps_ns = dps, d.p.take.count = dps ? e.ns[0] / dps : 0;
            d.p.take.total_ms_f = (float)(e.ns[0] / 1000000ull);
            d.p.take.fadeout = e.u32[0] ? 1u : 0u;
            return RB_OK;
        }
    }
}

static rb_status plan_stream(PlanStream& ps, uint16_t mixer_ch, uint32_t mixer_rate, std::vector<PlanStream>* all = nullptr, size_t self = 0) {
    const rb_stream_desc& d = ps.desc;
    ps.consumed = d.mix_start == RB_MIX_START_CONSUMED;
    ps.planning = true;
    {
        size_t n_app = 0;
        while (n_app < ps.fx.size() && ps.fx[n_app].kind == RB_FX_APPEND) n_app++;
        if (n_app) {
            if (!all) return fail(RB_ERR_UNSUPPORTED, "from_iter: the appended buffers are other descriptors of the batch (rb_batch_create)");
            auto seg_of = [](const rb_stream_desc& dd, SeqSeg& g) -> rb_status {
                if (dd.sample_rate == 0 || dd.channels == 0) return fail(RB_ERR_INVALID_ARGUMENT, "zero sample rate or channels");
                if (dd.channels > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "more than 12 channels");
                if (dd.format != RB_FMT_F32) return fail(RB_ERR_UNSUPPORTED, "from_iter: f32 buffers only");
                if (dd.span_len != 0 && (uint64_t)dd.span_len != dd.n_samples)
                    return fail(RB_ERR_UNSUPPORTED, "from_iter: span_len is n_samples (SamplesBuffer) or 0");
                g = SeqSeg{dd.n_samples, dd.channels, dd.sample_rate, dd.span_len != 0};
                return RB_OK;
            };
            std::vector<SeqSeg> segs(1);
            rb_status s0 = seg_of(d, segs[0]);
            if (s0 != RB_OK) return s0;
            for (size_t i = 0; i < n_app; i++) {
                const size_t idx = ps.fx[i].u32[0];
                if (idx >= all->size() || idx == self) return fail(RB_ERR_INVALID_ARGUMENT, "from_iter: bad index of an appended buffer");
                PlanStream& o = (*all)[idx];
                if (o.desc.mix_start != RB_MIX_START_CONSUMED || o.consumer >= 0 || o.planned || o.planning || !o.fx.empty())
                    return fail(RB_ERR_INVALID_ARGUMENT, "from_iter: an appended buffer is a descriptor without effects, mix_start = RB_MIX_START_CONSUMED, used once");
                SeqSeg g;
                rb_status so = seg_of(o.desc, g);
                if (so != RB_OK) return so;
                segs.push_back(g);
                o.consumer = (int64_t)self, o.appended_to = (int64_t)self, o.consumed = true, o.planned = true;
                ps.appended.push_back(idx);
            }
            for (const SeqSeg& g : segs) ps.seq_samples += g.n;
            return plan_varying(ps, segs, n_app, mixer_ch, mixer_rate);
        }
    }
    if (d.sample_rate == 0 || d.channels == 0) return fail(RB_ERR_INVALID_ARGUMENT, "zero sample rate or channels");
    if (d.channels > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "more than 12 channels");
    if (d.format > RB_FMT_I24_IN_I32) return fail(RB_ERR_INVALID_ARGUMENT, "unknown sample format");
    if (d.n_samples % d.channels != 0) return fail(RB_ERR_UNALIGNED_FRAMES, "n_samples % channels != 0");
    uint64_t n = d.n_samples;
    uint32_t c = d.channels, rate = d.sample_rate, span = d.span_len;
    const bool buffer_spans = d.span_len != 0 && (uint64_t)d.span_len == d.n_samples;   // SamplesBuffer semantics
    int64_t cv_last = -1;
    uint64_t tail_pad = 0;   // zeros a TakeDuration appended to complete its last frame (take.rs:113-123)
    if (d.format != RB_FMT_F32) {
        PlanNode nd;
        nd.d.kind = RB_N_CONVERT, nd.d.fmt = d.format, nd.d.c_in = nd.d.c_out = c, nd.d.n_in = nd.d.n_out = n;
        nd.rate_out = rate, nd.span_out = span;
        ps.nodes.push_back(nd);
    }
    bool first_fx = true;
    for (const rb_effect& e : ps.fx) {
        PlanNode nd;
        nd.d.c_in = nd.d.c_out = c, nd.d.n_in = nd.d.n_out = n;
        nd.rate_out = rate, nd.span_out = span;
        const bool is_first = first_fx;
        first_fx = false;
        switch (e.kind) {
            case RB_FX_MIX: {
                if (!all) return fail(RB_ERR_UNSUPPORTED, "mix: the second input is another descriptor of the batch (rb_batch_create)");
                const size_t idx = e.u32[0];
                if (idx >= all->size() || idx == self) return fail(RB_ERR_INVALID_ARGUMENT, "mix: bad index of the second input");
                PlanStream& o = (*all)[idx];
                if (o.desc.mix_start != RB_MIX_START_CONSUMED)
                    return fail(RB_ERR_INVALID_ARGUMENT, "mix: the second input must carry mix_start = RB_MIX_START_CONSUMED");
                if (o.consumer >= 0 || o.planning) return fail(RB_ERR_INVALID_ARGUMENT, "mix: the second input is consumed twice (or by itself)");
                if (!o.planned) {
                    rb_status so = plan_stream(o, mixer_ch, mixer_rate, all, idx);
                    if (so != RB_OK) return so;
                }
                o.consumer = (int64_t)self;
                // input1: UniformSourceIterator::new(self, channels, rate) (mix.rs:19) -- the identity on whole frames, but it never
                // pulls the frame padding of a TakeDuration and re-bootstraps per span like any other
                {
                    PlanNode u1;
                    rb_status s1 = plan_uniform(u1, (span && tail_pad) ? n - tail_pad : n, c, rate, span, c, rate, cv_last);
                    if (s1 != RB_OK) return s1;
                    if (u1.d.n_out != n) {
                        u1.level = ps.nodes.empty() ? 0u : ps.nodes.back().level + 1u;
                        ps.nodes.push_back(u1);
                        n = u1.d.n_out;
                    }
                }
                // input2: UniformSourceIterator::new(other, channels, rate) (mix.rs:20), appended to the OTHER stream's nodes
                uint64_t n2 = o.chain_len;
                {
                    PlanNode u2;
                    rb_status s2 = plan_uniform(u2, (o.end_span && o.end_tail_pad) ? o.chain_len - o.end_tail_pad : o.chain_len,
                                                o.chain_channels, o.chain_rate, o.end_span, c, rate, o.end_cv_last);
                    if (s2 != RB_OK) return s2;
                    if (!(u2.d.p.uni.from == u2.d.p.uni.to && u2.d.c_in == u2.d.c_out) || u2.d.n_out != o.chain_len) {
                        u2.level = o.nodes.empty() ? 0u : o.nodes.back().level + 1u;
                        o.nodes.push_back(u2);
                    }
                    n2 = u2.d.n_out;
                }
                nd.d.kind = RB_N_MIX2, nd.d.p.mix2.n2 = n2, nd.other = (int64_t)idx;
                nd.d.n_in = n, nd.d.n_out = std::max(n, n2);
                nd.span_out = 0;           // Mix::current_span_len of two UniformSourceIterators == None (mix.rs:80-88)
                nd.level = o.nodes.empty() ? 0u : o.nodes.back().level + 1u;
                cv_last = -1, tail_pad = 0;
                break;
            }
            case RB_FX_PAUSE: {
                // Pausable: while paused it hands out `channels` zeros per call round without pulling its input (pausable.rs:85-97);
                // a pause that would set in behind the source's last sample never does
                if (e.ns[0] > n || e.ns[1] == 0) continue;
                if (tail_pad) return fail(RB_ERR_UNSUPPORTED, "pause directly on a padded take_duration");
                nd.d.kind = RB_N_PAUSE, nd.d.p.pause.at = e.ns[0], nd.d.p.pause.n = e.ns[1] * c;
                nd.d.n_out = n + nd.d.p.pause.n;
                if (cv_last >= 0) cv_last = -1;
                break;
            }
            case RB_FX_SIGNAL: {
                // SignalGenerator::with_function (signal_generator.rs:107-128): mono, span-less, endless; `.take(n)` bounds it
                if (!is_first || d.n_samples != 0 || d.channels != 1 || d.format != RB_FMT_F32 || d.span_len != 0)
                    return fail(RB_ERR_INVALID_ARGUMENT, "signal generator: only as effects[0] of an empty mono f32 span-less descriptor");
                if (e.u32[0] > RB_SIGNAL_SAWTOOTH) return fail(RB_ERR_INVALID_ARGUMENT, "signal generator: unknown function");
                if (!(e.f32[0] > 0.0f)) return fail(RB_ERR_INVALID_ARGUMENT, "signal generator: frequency must be greater than zero");
                if (!std::isfinite(e.f32[0])) return fail(RB_ERR_UNSUPPORTED, "signal generator: infinite frequency");
                volatile float period = (float)rate / e.f32[0];          // :118
                nd.d.kind = RB_N_SIGNAL, nd.d.p.sig.step = 1.0f / period, nd.d.p.sig.fn = e.u32[0];   // :119
                nd.d.n_in = 0, nd.d.n_out = e.ns[0];
                break;
            }
            case RB_FX_AMPLIFY:
                nd.d.kind = RB_N_AMPLIFY, nd.d.p.amp.factor = e.f32[0];
                break;
            case RB_FX_SPEED:
                rate = rb_speed_sample_rate(rate, e.f32[0]);
                continue;   // metadata only
            case RB_FX_LOW_PASS:
            case RB_FX_HIGH_PASS: {
                hostmath::Blt k = hostmath::blt(e.kind == RB_FX_HIGH_PASS, e.u32[0], e.f32[0], rate);
                nd.d.kind = RB_N_BIQUAD;
                nd.d.p.blt = {k.b0, k.b1, k.b2, k.a1, k.a2};
                break;
            }
            case RB_FX_REVERB: {
                uint64_t D = rb_delay_samples(e.ns[0], rate, (uint16_t)c);
                nd.d.kind = RB_N_ECHO, nd.d.p.echo.delay = D, nd.d.p.echo.amplitude = e.f32[0];
                // Mix wraps both inputs in UniformSourceIterator (mix.rs:19-20): over a TakeDuration they never
                // pull the frame padding (see RB_FX_UNIFORM below)
                if (span && tail_pad) nd.d.n_in = n - tail_pad;
                nd.d.n_out = nd.d.n_in + D;
                cv_last = -1;
                tail_pad = 0;
                nd.span_out = 0;   // Mix::current_span_len of two UniformSourceIterators == None
                break;
            }
            case RB_FX_DELAY: {
                uint64_t D = rb_delay_samples(e.ns[0], rate, (uint16_t)c);
                if (span != 0 && (span < n || cv_last >= 0))
                    return fail(RB_ERR_UNSUPPORTED, "delay on a source with short spans");
                nd.d.kind = RB_N_DELAY, nd.d.p.echo.delay = D, nd.d.p.echo.amplitude = 1.0f;
                nd.d.n_out = n + D;
                if (span) nd.span_out = (uint32_t)std::min<uint64_t>((uint64_t)span + D, 0xFFFFFFFFull);
                break;
            }
            case RB_FX_AGC: {
                float mg = e.f32[1];
                if (!(mg >= 0.1f)) return fail(RB_ERR_INVALID_ARGUMENT, "agc: clamp(0.1, absolute_max_gain) would panic");
                uint64_t ten = 10ull * 1000000000ull;   // src/source/mod.rs:432-433
                nd.d.kind = RB_N_AGC;
                nd.d.p.agc.target = e.f32[0], nd.d.p.agc.max_gain = mg, nd.d.p.agc.floor = e.f32[2];
                nd.d.p.agc.attack = hostmath::duration_to_coefficient(std::min(e.ns[0], ten), rate);
                nd.d.p.agc.release = hostmath::duration_to_coefficient(std::min(e.ns[1], ten), rate);
                break;
            }
            case RB_FX_LIMIT: {
                nd.d.kind = RB_N_LIMIT;
                nd.d.p.lim = limit_params(e, rate);
                break;
            }
            case RB_FX_SPATIAL:
            case RB_FX_CHANNEL_VOLUME: {
                nd.d.kind = RB_N_CHANVOL;
                uint32_t co;
                if (e.kind == RB_FX_SPATIAL) {
                    co = 2;
                    hostmath::spatial_volumes(e.f32, e.f32 + 3, e.f32 + 6, nd.d.p.cv.vol);
                } else {
                    co = e.u32[0];
                    if (co == 0 || co > RB_MAX_CHANNELS) return fail(RB_ERR_INVALID_ARGUMENT, "channel_volume: 1..12 volumes");
                    for (uint32_t j = 0; j < co; j++) nd.d.p.cv.vol[j] = e.f32[j];
                }
                if (tail_pad) return fail(RB_ERR_UNSUPPORTED, "channel_volume/spatial directly on a padded take_duration");
                if (n % c != 0)
                    return fail(RB_ERR_UNALIGNED_FRAMES, "channel_volume/spatial on a stream that is not frame aligned "
                                                         "(e.g. after an odd-length delay)");
                nd.d.c_out = co;
                nd.d.n_out = (n / c) * co;
                cv_last = (buffer_spans && span != 0 && n >= c) ? (int64_t)((n / c - 1) * co) : -1;
                break;
            }
            case RB_FX_DISTORTION:
            case RB_FX_LINEAR_RAMP: {
                rb_status s = plan_pointwise(e, rate, c, nd.d);
                if (s != RB_OK) return s;
                break;
            }
            case RB_FX_TAKE_DURATION: {
                plan_pointwise(e, rate, c, nd.d);
                const uint64_t dps = nd.d.p.take.dps_ns;
                uint64_t take_n = dps ? nd.d.p.take.count : n;        // samples emitted before `remaining < dps`
                uint64_t count = std::min<uint64_t>(n, take_n);
                uint64_t pad = 0;
                if (dps && take_n <= n && count % c) pad = c - count % c;   // duration expired first: pad the frame
                nd.d.p.take.count = count;
                nd.d.n_out = count + pad;
                // a take that does not cut (it outlasts its input) hands the padding of a take INSIDE it on: the span it reports is still
                // the inner one's, so a UniformSourceIterator behind it stops in front of that padding all the same
                tail_pad = (dps && take_n >= n) ? tail_pad : pad;
                // TakeDuration::current_span_len: the inner span when it is shorter than what is left, else what is left
                uint64_t so = span ? std::min<uint64_t>(span, take_n) : take_n;
                nd.span_out = (uint32_t)std::min<uint64_t>(so, 0xFFFFFFFFull);
                if (nd.span_out == 0) nd.span_out = 1;   // Some(0) at the very end only; never None
                cv_last = -1;
                break;
            }
            case RB_FX_UNIFORM: {
                // a UniformSourceIterator over a TakeDuration asks for exactly the samples that are left
                // (take.rs:180-196), so the frame padding is never pulled
                rb_status s = plan_uniform(nd, (span && tail_pad) ? n - tail_pad : n, c, rate, span, e.u32[0], e.u32[1], cv_last);
                if (s != RB_OK) return s;
                cv_last = -1;
                tail_pad = 0;
                if (nd.d.p.uni.from == nd.d.p.uni.to && nd.d.c_in == nd.d.c_out && nd.d.n_out == n) {   // identity: no kernel
                    rate = nd.rate_out, span = 0;
                    continue;
                }
                break;
            }
            default: return fail(RB_ERR_INVALID_ARGUMENT, "unknown effect kind");
        }
        nd.level = std::max(nd.level, ps.nodes.empty() ? 0u : ps.nodes.back().level + 1u);
        ps.nodes.push_back(nd);
        n = nd.d.n_out, c = nd.d.c_out, rate = nd.rate_out, span = nd.span_out;
    }
    ps.chain_len = n, ps.chain_channels = c, ps.chain_rate = rate;
    ps.end_span = span, ps.end_tail_pad = tail_pad, ps.end_cv_last = cv_last;
    ps.planning = false, ps.planned = true;
    if (ps.consumed) {   // the MIX that consumes it appends the conversion to ITS format; the mixer never sees this stream
        ps.out_len = 0, ps.mix_start = 0;
        return RB_OK;
    }
    // Mixer::add wraps the source in UniformSourceIterator::new(source, mixer_ch, mixer_rate) (mixer.rs:62-63)
    {
        PlanNode nd;
        rb_status s = plan_uniform(nd, (span && tail_pad) ? n - tail_pad : n, c, rate, span, mixer_ch, mixer_rate, cv_last);
        if (s != RB_OK) return s;
        if (!(nd.d.p.uni.from == nd.d.p.uni.to && nd.d.c_in == nd.d.c_out) || nd.d.n_out != n) {
            nd.level = ps.nodes.empty() ? 0u : ps.nodes.back().level + 1u;
            ps.nodes.push_back(nd);
            n = nd.d.n_out;
        }
    }
    ps.out_len = n;
    // start_pending_sources: a source joins at the next frame boundary (mixer.rs:175-183)
    ps.mix_start = (d.mix_start + mixer_ch - 1) / mixer_ch * mixer_ch;
    return RB_OK;
}

extern "C" rb_status rb_stream_plan(const rb_stream_desc* desc, uint16_t mixer_ch, uint32_t mixer_rate,
                                    uint64_t* out_len, uint16_t* chain_channels, uint32_t* chain_rate,
                                    uint64_t* chain_len) {
    if (!desc) return fail(RB_ERR_INVALID_ARGUMENT, "desc is NULL");
    if (mixer_ch == 0 || mixer_rate == 0) return fail(RB_ERR_INVALID_ARGUMENT, "mixer: zero channels or rate");
    if (mixer_ch > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "mixer: more than 12 channels");
    if (desc->n_effects && !desc->effects) return fail(RB_ERR_INVALID_ARGUMENT, "effects is NULL");
    PlanStream ps;
    ps.desc = *desc;
    ps.fx.assign(desc->effects, desc->effects + desc->n_effects);
    rb_status s = plan_stream(ps, mixer_ch, mixer_rate);
    if (s != RB_OK) return s;
    if (out_len) *out_len = ps.out_len;
    if (chain_channels) *chain_channels = (uint16_t)ps.chain_channels;
    if (chain_rate) *chain_rate = ps.chain_rate;
    if (chain_len) *chain_len = ps.chain_len;
    return RB_OK;
}

// The same closed forms for descriptor `stream` of an array -- needed when a descriptor names others (RB_FX_MIX, RB_FX_APPEND).
extern "C" rb_status rb_streams_plan(const rb_stream_desc* descs, size_t n_streams, size_t stream, uint16_t mixer_ch, uint32_t mixer_rate,
                                     uint64_t* out_len, uint16_t* chain_channels, uint32_t* chain_rate, uint64_t* chain_len) {
    if (!descs || stream >= n_streams) return fail(RB_ERR_INVALID_ARGUMENT, "descs is NULL or stream out of range");
    if (mixer_ch == 0 || mixer_rate == 0) return fail(RB_ERR_INVALID_ARGUMENT, "mixer: zero channels or rate");
    if (mixer_ch > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "mixer: more than 12 channels");
    std::vector<PlanStream> all(n_streams);
    for (size_t i = 0; i < n_streams; i++) {
        if (descs[i].n_effects && !descs[i].effects) return fail(RB_ERR_INVALID_ARGUMENT, "effects is NULL");
        all[i].desc = descs[i];
        all[i].fx.assign(descs[i].effects, descs[i].effects + descs[i].n_effects);
    }
    for (size_t i = 0; i < n_streams; i++) {
        if (all[i].planned) continue;
        rb_status s = plan_stream(all[i], mixer_ch, mixer_rate, &all, i);
        if (s != RB_OK) return s;
    }
    const PlanStream& ps = all[stream];
    if (out_len) *out_len = ps.out_len;
    if (chain_channels) *chain_channels = (uint16_t)ps.chain_channels;
    if (chain_rate) *chain_rate = ps.chain_rate;
    if (chain_len) *chain_len = ps.chain_len;
    return RB_OK;
}

// ------------------------------------------------------------------------------------------------
// batch
// ------------------------------------------------------------------------------------------------
struct LaunchGroup {
    uint32_t kind;
    uint32_t first, count;   // range in d_nodes
    uint64_t max_n_out;
    uint32_t max_channels;
};
struct rb_batch {
    rb_context* ctx = nullptr;
    uint16_t mixer_ch = 0;
    uint32_t mixer_rate = 0;
    uint32_t flags = 0;
    std::vector<PlanStream> streams;
    uint64_t mix_len = 0;
    uint64_t algo_bytes = 0;
    // device memory
    uint8_t* d_in = nullptr;
    size_t in_bytes = 0;
    float* d_buf[2] = {nullptr, nullptr};
    float* d_aux[2] = {nullptr, nullptr};   // scratch rows for multi-pass adapters (AGC)
    size_t buf_floats = 0;
    rb_node_dev* d_nodes = nullptr;
    rb_mix_src* d_mix = nullptr;
    float* d_mix_partial = nullptr;   // [mix_groups][mix_len] when the source list is summed in concurrent runs
    uint32_t mix_groups = 1;
    float* d_out = nullptr;
    std::vector<LaunchGroup> groups;
    rb_fused_plan* fused = nullptr;   // non-null when the fused path serves this batch
    // Integer PCM (what decoders yield: src/decoder/wav.rs:119-151) in front of a fused plan: the batch keeps an f32 copy of the
    // inputs resident (SampleTypeConverter, src/conversions/sample.rs:42-44, applied once per upload by k_convert), the fused
    // kernels read that -- the host -> device copy moves 2 bytes per sample instead of 4.
    float* d_in_f32 = nullptr;
    rb_node_dev* d_conv_nodes = nullptr;   // one RB_N_CONVERT record per stream: raw arena -> f32 arena
    uint64_t conv_max_n = 0;
    bool conv_dirty = false;               // raw inputs were (re)written since the last conversion
    uint32_t launches = 0;
    bool rendered = false;
    std::vector<uint8_t> uploaded;
    // adapters on the MixerSource (rb_batch_set_master), run in place on d_out behind the mix
    std::vector<rb_master_run> master_runs;   // the active runs of the mix, known from the closed-form lengths
    uint64_t master_seq = 0;                  // samples in them
    bool runs_aligned = true;                 // every run ends on a frame boundary
    bool has_master = false;
    rb_master_params master{};
    rb_master_run* d_master_runs = nullptr;
};

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" rb_status rb_batch_destroy(rb_batch* b) {
    if (!b) return RB_OK;
    cudaSetDevice(b->ctx->device);
    cudaStreamSynchronize(b->ctx->stream);
    if (b->fused) rb_fused_destroy(b->fused);
    cudaFree(b->d_in);
    cudaFree(b->d_in_f32);
    cudaFree(b->d_conv_nodes);
    cudaFree(b->d_buf[0]);
    cudaFree(b->d_buf[1]);
    cudaFree(b->d_aux[0]);
    cudaFree(b->d_aux[1]);
    cudaFree(b->d_nodes);
    cudaFree(b->d_mix);
    cudaFree(b->d_mix_partial);
    cudaFree(b->d_out);
    cudaFree(b->d_master_runs);
    delete b;
    return RB_OK;
}

extern "C" rb_status rb_batch_create(rb_context* ctx, uint16_t mixer_ch, uint32_t mixer_rate,
                                     const rb_stream_desc* descs, size_t n_streams, uint32_t flags, rb_batch** out) {
    if (!ctx || !out || (!descs && n_streams)) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (mixer_ch == 0 || mixer_rate == 0) return fail(RB_ERR_INVALID_ARGUMENT, "mixer: zero channels or rate");
    if (mixer_ch > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "mixer: more than 12 channels");
    if (n_streams > 0x7FFFFFFFull) return fail(RB_ERR_UNSUPPORTED, "too many streams");
    RB_CUDA(cudaSetDevice(ctx->device));
    std::unique_ptr<rb_batch, rb_status (*)(rb_batch*)> b(new (std::nothrow) rb_batch, rb_batch_destroy);
    if (!b) return fail(RB_ERR_OUT_OF_MEMORY, "host allocation failed");
    b->ctx = ctx, b->mixer_ch = mixer_ch, b->mixer_rate = mixer_rate, b->flags = flags;
    b->streams.resize(n_streams);
    b->uploaded.assign(n_streams, 0);
    size_t in_bytes = 0, buf_floats = 0;
    uint64_t mix_len = 0, algo = 0;
    bool any_consumed = false;
    for (size_t i = 0; i < n_streams; i++) {
        PlanStream& ps = b->streams[i];
        ps.desc = descs[i];
        if (descs[i].n_effects && !descs[i].effects) return fail(RB_ERR_INVALID_ARGUMENT, "effects is NULL");
        ps.fx.assign(descs[i].effects, descs[i].effects + descs[i].n_effects);
        ps.desc.effects = nullptr;
        any_consumed = any_consumed || descs[i].mix_start == RB_MIX_START_CONSUMED;
    }
    for (size_t i = 0; i < n_streams; i++) {
        PlanStream& ps = b->streams[i];
        if (ps.planned) continue;   // the second input of a MIX further up: planned when that MIX was reached
        rb_status s = plan_stream(ps, mixer_ch, mixer_rate, &b->streams, i);
        if (s != RB_OK) {
            g_last_error = "stream " + std::to_string(i) + ": " + g_last_error;
            return s;
        }
    }
    uint32_t max_level = 0;
    for (size_t i = 0; i < n_streams; i++) {
        PlanStream& ps = b->streams[i];
        if (ps.consumed && ps.consumer < 0)
            return fail(RB_ERR_INVALID_ARGUMENT, "stream " + std::to_string(i) + ": mix_start = RB_MIX_START_CONSUMED but no RB_FX_MIX names it");
        if (ps.appended_to < 0) {   // the buffers of a from_iter sequence follow their head without a gap
            ps.in_off = in_bytes;
            size_t off = in_bytes + (size_t)ps.desc.n_samples * fmt_size(ps.desc.format);
            for (size_t idx : ps.appended) {
                b->streams[idx].in_off = off;
                off += (size_t)b->streams[idx].desc.n_samples * sizeof(float);
            }
            in_bytes = align_up(off + 16, 128);
        }
        uint64_t cap = 0;
        for (auto& nd : ps.nodes) cap = std::max(cap, nd.d.n_out), max_level = std::max(max_level, nd.level + 1u);
        if (!ps.runs.empty()) cap = std::max(cap, ps.out_len), max_level = std::max(max_level, ps.run_level + 1u);
        ps.buf_cap = align_up((size_t)cap + 4, 32);
        ps.buf_off = buf_floats;
        buf_floats += ps.buf_cap;
        if (ps.out_len) mix_len = std::max(mix_len, ps.mix_start + ps.out_len);
        algo += ps.desc.n_samples * fmt_size(ps.desc.format);
    }
    b->mix_len = mix_len;
    b->algo_bytes = algo + mix_len * 4;
    {   // active runs: MixerSource::next() is Some where a source plays (mixer.rs:120-136); the gaps between are written as 0.0
        std::vector<std::pair<uint64_t, uint64_t>> iv;
        for (const PlanStream& ps : b->streams)
            if (ps.out_len && !ps.consumed && ps.appended_to < 0) iv.push_back({ps.mix_start, ps.mix_start + ps.out_len});
        std::sort(iv.begin(), iv.end());
        uint64_t seq = 0;
        for (size_t i = 0; i < iv.size();) {
            uint64_t lo = iv[i].first, hi = iv[i].second;
            for (i++; i < iv.size() && iv[i].first <= hi; i++) hi = std::max(hi, iv[i].second);
            b->runs_aligned = b->runs_aligned && lo % mixer_ch == 0 && hi % mixer_ch == 0;
            b->master_runs.push_back({seq + (hi - lo), lo - seq});
            seq += hi - lo;
        }
        b->master_seq = seq;
    }
    b->in_bytes = in_bytes;

    RB_CUDA(cudaMalloc(&b->d_in, std::max<size_t>(in_bytes, 256)));
    RB_CUDA(cudaMalloc(&b->d_out, std::max<size_t>(mix_len * 4, 256)));

    // Mixer insertion order: Mixer::add calls arrive in increasing output position, ties in array order
    // (src/mixer.rs:175-183 appends pending sources in arrival order) -> stable sort by mix_start.
    std::vector<size_t> order(n_streams);
    std::iota(order.begin(), order.end(), (size_t)0);
    std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) {
        return b->streams[x].desc.mix_start < b->streams[y].desc.mix_start;
    });

    // Fast path: one fused kernel family when the whole batch has a chain shape it understands.
    if (!(flags & RB_NO_FUSION) && !any_consumed) {   // a two-input MIX: general path
        std::vector<rb_fused_stream> fs(n_streams);
        bool ok = true;
        // every stream integer PCM: plan the fused kernels on a resident f32 copy (converted once per upload)
        bool all_int = n_streams > 0;
        for (size_t i = 0; i < n_streams; i++) all_int = all_int && b->streams[i].desc.format != RB_FMT_F32 && !b->streams[i].nodes.empty();
        std::vector<size_t> f32_off(n_streams, 0);
        if (all_int) {
            size_t floats = 0;
            for (size_t i = 0; i < n_streams; i++) f32_off[i] = floats, floats += align_up((size_t)b->streams[i].desc.n_samples + 4, 32);
            RB_CUDA(cudaMalloc(&b->d_in_f32, std::max<size_t>(floats * sizeof(float), 256)));
            RB_CUDA(cudaMemsetAsync(b->d_in_f32, 0, std::max<size_t>(floats * sizeof(float), 256), ctx->stream));
        }
        for (size_t i = 0; i < n_streams && ok; i++) {
            PlanStream& ps = b->streams[order[i]];
            fs[i].in = all_int ? (const void*)(b->d_in_f32 + f32_off[order[i]]) : (const void*)(b->d_in + ps.in_off);
            fs[i].fmt = all_int ? (uint32_t)RB_FMT_F32 : ps.desc.format;
            fs[i].n_nodes = (uint32_t)ps.nodes.size() - (all_int ? 1u : 0u);
            fs[i].nodes = fs[i].n_nodes == 0 ? nullptr : &ps.nodes[all_int ? 1 : 0].d;
            fs[i].node_stride = sizeof(PlanNode);
            fs[i].out_len = ps.out_len;
            fs[i].mix_start = ps.mix_start;
            fs[i].n_in = ps.desc.n_samples;
            fs[i].c_in = ps.desc.channels;
        }
        if (ok) {
            rb_fused_plan* fp = nullptr;
            cudaError_t e = rb_fused_try_create(fs.data(), n_streams, mixer_ch, b->d_out, mix_len, flags,
                                                ctx->sm_count, ctx->stream, &fp);
            if (e != cudaSuccess) return fail(RB_ERR_CUDA, std::string("fused plan: ") + cudaGetErrorString(e));
            b->fused = fp;   // may be null: shape not covered -> general path
        }
        if (all_int && b->fused) {
            std::vector<rb_node_dev> conv(n_streams);
            for (size_t i = 0; i < n_streams; i++) {
                const PlanStream& ps = b->streams[i];
                rb_node_dev nd = ps.nodes[0].d;          // the RB_N_CONVERT the planner put in front
                nd.src = b->d_in + ps.in_off, nd.dst = b->d_in_f32 + f32_off[i];
                conv[i] = nd;
                b->conv_max_n = std::max(b->conv_max_n, nd.n_out);
            }
            RB_CUDA(cudaMalloc(&b->d_conv_nodes, n_streams * sizeof(rb_node_dev)));
            RB_CUDA(cudaMemcpy(b->d_conv_nodes, conv.data(), n_streams * sizeof(rb_node_dev), cudaMemcpyHostToDevice));
            b->conv_dirty = true;
        } else if (all_int) {
            cudaFree(b->d_in_f32);
            b->d_in_f32 = nullptr;
            // no fused kernel took the f32 view: plan again on the raw format (the generic fused kernels convert at load time)
            for (size_t i = 0; i < n_streams; i++) {
                PlanStream& ps = b->streams[order[i]];
                fs[i].in = b->d_in + ps.in_off, fs[i].fmt = ps.desc.format;
                fs[i].n_nodes = (uint32_t)ps.nodes.size(), fs[i].nodes = &ps.nodes[0].d;
            }
            rb_fused_plan* fp = nullptr;
            cudaError_t e = rb_fused_try_create(fs.data(), n_streams, mixer_ch, b->d_out, mix_len, flags, ctx->sm_count, ctx->stream, &fp);
            if (e != cudaSuccess) return fail(RB_ERR_CUDA, std::string("fused plan: ") + cudaGetErrorString(e));
            b->fused = fp;
        }
    }

    if (!b->fused || (flags & RB_KEEP_STREAM_OUTPUTS)) {
        // general path: two ping-pong arenas, one kernel per adapter level and kind
        b->buf_floats = buf_floats;
        RB_CUDA(cudaMalloc(&b->d_buf[0], std::max<size_t>(buf_floats * 4, 256)));
        RB_CUDA(cudaMalloc(&b->d_buf[1], std::max<size_t>(buf_floats * 4, 256)));
        bool need_aux = false;
        for (auto& ps : b->streams)
            for (auto& nd : ps.nodes) need_aux = need_aux || nd.d.kind == RB_N_AGC;
        if (need_aux) {
            RB_CUDA(cudaMalloc(&b->d_aux[0], std::max<size_t>(buf_floats * 4, 256)));
            RB_CUDA(cudaMalloc(&b->d_aux[1], std::max<size_t>(buf_floats * 4, 256)));
        }
        std::vector<rb_node_dev> host_nodes;
        auto final_of = [&](const PlanStream& ps) -> const float* {
            const size_t k = ps.nodes.size() + (ps.runs.empty() ? 0 : 1);   // the converter runs of a from_iter source count as one node
            return (k == 0) ? (const float*)(b->d_in + ps.in_off) : b->d_buf[(k - 1) & 1] + ps.buf_off;
        };
        for (uint32_t lvl = 0; lvl < max_level; lvl++) {
            for (uint32_t kind = 0; kind < RB_N_KINDS; kind++) {
                LaunchGroup g{kind, (uint32_t)host_nodes.size(), 0, 0, 0};
                for (auto& ps : b->streams) {
                    for (size_t j = 0; j < ps.nodes.size(); j++) {   // node j reads arena (j-1)&1 and writes arena j&1, at launch level `level`
                        if (ps.nodes[j].level != lvl || ps.nodes[j].d.kind != kind) continue;
                        rb_node_dev nd = ps.nodes[j].d;
                        nd.src = (j == 0) ? (const void*)(b->d_in + ps.in_off)
                                          : (const void*)(b->d_buf[(j - 1) & 1] + ps.buf_off);
                        nd.dst = b->d_buf[j & 1] + ps.buf_off;
                        nd.aux0 = b->d_aux[0] ? b->d_aux[0] + ps.buf_off : nullptr;
                        nd.aux1 = b->d_aux[1] ? b->d_aux[1] + ps.buf_off : nullptr;
                        if (kind == RB_N_MIX2) nd.aux0 = const_cast<float*>(final_of(b->streams[(size_t)ps.nodes[j].other]));
                        if (!ps.nodes[j].splits.empty()) {
                            // from_iter: the adapter starts from scratch at a span boundary -- one node per run of samples
                            for (const PlanNode::Split& sp : ps.nodes[j].splits) {
                                if (sp.n == 0) continue;
                                rb_node_dev r = sp.d;
                                r.src = (const float*)nd.src + sp.off, r.dst = nd.dst + sp.off;
                                r.aux0 = nd.aux0 ? nd.aux0 + sp.off : nullptr, r.aux1 = nd.aux1 ? nd.aux1 + sp.off : nullptr;
                                r.n_in = r.n_out = sp.n;
                                host_nodes.push_back(r);
                                g.count++;
                                g.max_n_out = std::max(g.max_n_out, r.n_out);
                                g.max_channels = std::max(g.max_channels, r.c_in);
                            }
                            continue;
                        }
                        host_nodes.push_back(nd);
                        g.count++;
                        g.max_n_out = std::max(g.max_n_out, nd.n_out);
                        g.max_channels = std::max(g.max_channels, nd.c_in);
                    }
                    if (kind == RB_N_UNIFORM && !ps.runs.empty() && ps.run_level == lvl) {
                        // from_iter: one k_uniform node per converter run, each on its slice of the sequence, outputs back to back
                        const size_t j = ps.nodes.size();
                        const float* in = (j == 0) ? (const float*)(b->d_in + ps.in_off) : b->d_buf[(j - 1) & 1] + ps.buf_off;
                        for (const PlanStream::Run& run : ps.runs) {
                            rb_node_dev nd = run.nd.d;
                            nd.src = in + run.in_off, nd.dst = b->d_buf[j & 1] + ps.buf_off + run.out_off;
                            nd.aux0 = nd.aux1 = nullptr;
                            host_nodes.push_back(nd);
                            g.count++;
                            g.max_n_out = std::max(g.max_n_out, nd.n_out);
                            g.max_channels = std::max(g.max_channels, nd.c_in);
                        }
                    }
                }
                if (g.count) b->groups.push_back(g);
            }
        }
        RB_CUDA(cudaMalloc(&b->d_nodes, std::max<size_t>(host_nodes.size() * sizeof(rb_node_dev), 256)));
        if (!host_nodes.empty())
            RB_CUDA(cudaMemcpy(b->d_nodes, host_nodes.data(), host_nodes.size() * sizeof(rb_node_dev),
                               cudaMemcpyHostToDevice));
        std::vector<rb_mix_src> mix(n_streams);
        for (size_t i = 0; i < n_streams; i++) {
            PlanStream& ps = b->streams[order[i]];
            ps.final_ptr = final_of(ps);
            mix[i] = {ps.final_ptr, ps.mix_start, ps.out_len};
        }
        RB_CUDA(cudaMalloc(&b->d_mix, std::max<size_t>(n_streams * sizeof(rb_mix_src), 256)));
        if (n_streams)
            RB_CUDA(cudaMemcpy(b->d_mix, mix.data(), n_streams * sizeof(rb_mix_src), cudaMemcpyHostToDevice));
        // Few output samples, many sources (short blocks of a big mixer): one thread per four outputs leaves most SMs
        // idle.  Unless the caller pinned the summation order, cut the source list into runs summed concurrently.
        const uint64_t mix_blocks = ((mix_len + 3) / 4 + 255) / 256;
        const uint64_t want_blocks = 2ull * (uint64_t)ctx->sm_count;
        if (!(flags & RB_MIX_EXACT_ORDER) && mix_len && n_streams >= 256 && mix_blocks < want_blocks) {
            uint64_t g = (want_blocks + mix_blocks - 1) / mix_blocks;
            g = std::min<uint64_t>(g, n_streams / 64);
            g = std::min<uint64_t>(g, 64);
            if (g > 1) {
                RB_CUDA(cudaMalloc(&b->d_mix_partial, (size_t)g * ((mix_len + 3) & ~3ull) * sizeof(float)));
                b->mix_groups = (uint32_t)g;
            }
        }
    }
    uint32_t general_launches = 0;
    for (const LaunchGroup& g : b->groups) general_launches += (g.kind == RB_N_AGC) ? 3u : 1u;
    b->launches = b->fused ? rb_fused_launch_count(b->fused) : general_launches + (mix_len ? (b->mix_groups > 1 ? 2u : 1u) : 0u);
    if (b->fused && (flags & RB_KEEP_STREAM_OUTPUTS)) b->launches += general_launches;
    *out = b.release();
    return RB_OK;
}

static rb_status check_stream(rb_batch* b, size_t stream) {
    if (!b) return fail(RB_ERR_INVALID_ARGUMENT, "batch is NULL");
    if (stream >= b->streams.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    return RB_OK;
}

extern "C" rb_status rb_batch_upload(rb_batch* b, size_t stream, const void* pcm, uint64_t n_samples) {
    rb_status s = check_stream(b, stream);
    if (s != RB_OK) return s;
    PlanStream& ps = b->streams[stream];
    if (n_samples != ps.desc.n_samples) return fail(RB_ERR_INVALID_ARGUMENT, "n_samples differs from the descriptor");
    if (!pcm && n_samples) return fail(RB_ERR_INVALID_ARGUMENT, "pcm is NULL");
    RB_CUDA(cudaSetDevice(b->ctx->device));
    if (n_samples)
        RB_CUDA(cudaMemcpyAsync(b->d_in + ps.in_off, pcm, n_samples * fmt_size(ps.desc.format), cudaMemcpyHostToDevice,
                                b->ctx->stream));
    b->uploaded[stream] = 1;
    b->conv_dirty = true;
    rb_fused_inputs_changed(b->fused);
    return RB_OK;
}

extern "C" rb_status rb_batch_upload_packed(rb_batch* b, const void* pcm, uint64_t total_samples) {
    if (!b || (!pcm && total_samples)) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    uint64_t tot = 0;
    for (auto& ps : b->streams) tot += ps.desc.n_samples;
    if (tot != total_samples) return fail(RB_ERR_INVALID_ARGUMENT, "total_samples differs from the descriptors");
    RB_CUDA(cudaSetDevice(b->ctx->device));
    const uint8_t* p = (const uint8_t*)pcm;
    // Streams with equal byte sizes are laid out with a constant device pitch: one strided 2-D copy
    // instead of one cudaMemcpyAsync per stream.
    size_t i = 0, n = b->streams.size();
    while (i < n) {
        size_t bytes = (size_t)b->streams[i].desc.n_samples * fmt_size(b->streams[i].desc.format);
        size_t j = i + 1;
        // (the buffers of a from_iter sequence sit inside their head's region: only ascending, non-overlapping offsets form a pitch)
        size_t pitch = (j < n && b->streams[j].in_off >= b->streams[i].in_off + bytes) ? b->streams[j].in_off - b->streams[i].in_off : 0;
        while (pitch && j < n && (size_t)b->streams[j].desc.n_samples * fmt_size(b->streams[j].desc.format) == bytes &&
               b->streams[j].in_off > b->streams[j - 1].in_off && b->streams[j].in_off - b->streams[j - 1].in_off == pitch)
            j++;
        size_t rows = j - i;
        if (bytes) {
            if (rows > 1)
                RB_CUDA(cudaMemcpy2DAsync(b->d_in + b->streams[i].in_off, pitch, p, bytes, bytes, rows,
                                          cudaMemcpyHostToDevice, b->ctx->stream));
            else
                RB_CUDA(cudaMemcpyAsync(b->d_in + b->streams[i].in_off, p, bytes, cudaMemcpyHostToDevice,
                                        b->ctx->stream));
        }
        p += bytes * rows;
        for (size_t k = i; k < j; k++) b->uploaded[k] = 1;
        i = j;
    }
    b->conv_dirty = true;
    rb_fused_inputs_changed(b->fused);
    return RB_OK;
}

extern "C" rb_status rb_batch_input_device_ptr(rb_batch* b, size_t stream, void** dptr, uint64_t* capacity) {
    rb_status s = check_stream(b, stream);
    if (s != RB_OK) return s;
    if (!dptr) return fail(RB_ERR_INVALID_ARGUMENT, "dptr is NULL");
    PlanStream& ps = b->streams[stream];
    *dptr = b->d_in + ps.in_off;
    if (capacity) *capacity = ps.desc.n_samples;
    b->uploaded[stream] = 1;   // the caller takes responsibility for the contents
    b->conv_dirty = true;
    rb_fused_inputs_changed(b->fused);   // ... and asks for the pointer again after rewriting them
    return RB_OK;
}

extern "C" rb_status rb_batch_stream_out_len(rb_batch* b, size_t stream, uint64_t* n) {
    rb_status s = check_stream(b, stream);
    if (s != RB_OK) return s;
    if (!n) return fail(RB_ERR_INVALID_ARGUMENT, "n is NULL");
    *n = b->streams[stream].out_len;
    return RB_OK;
}
extern "C" rb_status rb_batch_mix_len(rb_batch* b, uint64_t* n) {
    if (!b || !n) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *n = b->mix_len;
    return RB_OK;
}
extern "C" rb_status rb_batch_launches_per_render(rb_batch* b, uint32_t* n) {
    if (!b || !n) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *n = b->launches + (b->has_master && b->master_seq ? 1u : 0u);
    return RB_OK;
}
extern "C" rb_status rb_batch_set_master(rb_batch* b, const rb_effect* effects, uint32_t n_effects) {
    if (!b) return fail(RB_ERR_INVALID_ARGUMENT, "batch is NULL");
    rb_master_params p{};
    rb_status s = parse_master(effects, n_effects, b->mixer_rate, &p);
    if (s != RB_OK) return s;
    if (n_effects == 0) {
        b->has_master = false;
        return RB_OK;
    }
    // Limit::next keeps its channel position across a gap (it is not pulled there): a run that ends inside a frame would
    // shift every later frame's channels, which the kernel's frame tiles do not follow
    if (!b->runs_aligned)
        return fail(RB_ERR_UNALIGNED_FRAMES, "master chain: an active run of the mix ends inside a frame (a chain with a trailing partial frame)");
    if (!b->d_master_runs && !b->master_runs.empty()) {
        RB_CUDA(cudaSetDevice(b->ctx->device));
        RB_CUDA(cudaMalloc(&b->d_master_runs, b->master_runs.size() * sizeof(rb_master_run)));
        RB_CUDA(cudaMemcpy(b->d_master_runs, b->master_runs.data(), b->master_runs.size() * sizeof(rb_master_run), cudaMemcpyHostToDevice));
    }
    b->master = p, b->has_master = true;
    return RB_OK;
}
extern "C" rb_status rb_batch_kernel_family(rb_batch* b, int* family) {
    if (!b || !family) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *family = b->fused ? rb_fused_kind(b->fused) : -1;
    return RB_OK;
}
extern "C" rb_status rb_batch_mix_group(rb_batch* b, uint32_t* rows) {
    if (!b || !rows) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *rows = b->fused ? rb_fused_mix_group(b->fused) : 0u;
    return RB_OK;
}
extern "C" rb_status rb_batch_algorithmic_bytes(rb_batch* b, uint64_t* bytes) {
    if (!b || !bytes) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *bytes = b->algo_bytes;
    return RB_OK;
}

static rb_status run_general(rb_batch* b, bool with_mix) {
    cudaStream_t st = b->ctx->stream;
    for (const LaunchGroup& g : b->groups)
        RB_CUDA(rb_launch_nodes(g.kind, b->d_nodes + g.first, g.count, g.max_n_out, g.max_channels, st));
    if (with_mix)
        RB_CUDA(rb_launch_mix(b->d_mix, (uint32_t)b->streams.size(), b->d_out, b->mix_len, st, b->d_mix_partial, b->mix_groups));
    return RB_OK;
}

static rb_status render_device(rb_batch* b, bool skip_final_sum);
extern "C" rb_status rb_batch_render_mix_device(rb_batch* b) { return render_device(b, false); }
// skip_final_sum: the fused plan's last launch (the ordered sum of its per-CTA partial rows) is left to the caller (rb_p2p)
static rb_status render_device(rb_batch* b, bool skip_final_sum) {
    if (!b) return fail(RB_ERR_INVALID_ARGUMENT, "batch is NULL");
    for (size_t i = 0; i < b->streams.size(); i++)
        if (!b->uploaded[i] && b->streams[i].desc.n_samples)
            return fail(RB_ERR_STATE, "stream " + std::to_string(i) + " was never uploaded");
    RB_CUDA(cudaSetDevice(b->ctx->device));
    if (b->fused) {
        if (b->d_conv_nodes && b->conv_dirty) {   // integer PCM was uploaded: refresh the resident f32 copy
            RB_CUDA(rb_launch_nodes(RB_N_CONVERT, b->d_conv_nodes, (uint32_t)b->streams.size(), b->conv_max_n, 1, b->ctx->stream));
            b->conv_dirty = false;
        }
        RB_CUDA(rb_fused_run(b->fused, b->ctx->stream, skip_final_sum));
        if (b->flags & RB_KEEP_STREAM_OUTPUTS) {
            rb_status s = run_general(b, false);
            if (s != RB_OK) return s;
        }
    } else {
        rb_status s = run_general(b, true);
        if (s != RB_OK) return s;
    }
    if (b->has_master)
        RB_CUDA(rb_launch_master(b->d_out, b->d_master_runs, (uint32_t)b->master_runs.size(), b->master_seq, b->mixer_ch, b->master, nullptr,
                                 nullptr, b->ctx->stream));
    b->rendered = true;
    return RB_OK;
}
// ----------------------------------------------------------------------------------------------------
// Multi-GPU: the cross-shard mixer sum (SURVEY.md 8b/8e).  Streams are independent until the mixer adds them
// (src/mixer.rs:185-198), so every GPU renders the partial mix of its own shard and ONE all-reduce(sum, f32, mix_len)
// gives every rank the MixerSource output.  The collective is NCCL's (over NVLink / NVSwitch on an H100 node), called
// from here on the context's stream, so a Rust / C host needs no NCCL binding of its own.  The library is loaded on first
// use (dlopen "libnccl.so.2": a process that already holds NCCL -- torch -- shares that copy); a build without NCCL on the
// box fails the call loudly, nothing falls back to the host.
// ----------------------------------------------------------------------------------------------------
#include <dlfcn.h>
namespace {
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, rb_comm_id, int) = nullptr;
    int (*CommInitAll)(void**, int, const int*) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
NcclApi* nccl_api(std::string* why) {
    static NcclApi api;
    static bool tried = false;
    static std::string err;
    if (!tried) {
        tried = true;
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
            api.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) err = std::string("cannot load libnccl.so.2: ") + (dlerror() ? dlerror() : "?");
        else {
            auto sym = [&](const char* n) {
                void* p = dlsym(api.lib, n);
                if (!p && err.empty()) err = std::string("libnccl lacks ") + n;
                return p;
            };
            api.GetUniqueId = (int (*)(void*))sym("ncclGetUniqueId");
            api.CommInitRank = (int (*)(void**, int, rb_comm_id, int))sym("ncclCommInitRank");
            api.CommInitAll = (int (*)(void**, int, const int*))sym("ncclCommInitAll");
            api.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))sym("ncclAllReduce");
            api.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))sym("ncclAllGather");
            api.CommDestroy = (int (*)(void*))sym("ncclCommDestroy");
            api.GroupStart = (int (*)())sym("ncclGroupStart");
            api.GroupEnd = (int (*)())sym("ncclGroupEnd");
            api.GetErrorString = (const char* (*)(int))sym("ncclGetErrorString");
        }
    }
    if (!err.empty()) {
        if (why) *why = err;
        return nullptr;
    }
    return &api;
}
constexpr int NCCL_FLOAT32 = 7, NCCL_SUM = 0, NCCL_INT8 = 0;   // ncclFloat32, ncclSum, ncclInt8 (nccl.h)
}  // namespace

struct rb_comm {
    std::vector<void*> comms;           // one per local rank (one entry for the process-per-GPU form)
    std::vector<rb_context*> ctxs;
    int n_ranks = 0;
    int rank = 0;                       // process-per-GPU form
    // the mixes are exchanged by k_mix_exchange over NVLink peer memory (rb_p2p.h) where the ranks can map each other's
    // mailboxes; NCCL's all-reduce otherwise (other nodes, IPC not permitted, RB_COMM_NCCL_ONLY=1).  Set up at the first call.
    std::vector<rb_p2p*> p2p;           // one per local rank, or empty
    bool p2p_tried = false;
    std::string transport = "nccl (ncclAllReduce sum f32 on the render stream)";
};

#define RB_NCCL(call, api)                                                                             \
    do {                                                                                               \
        const int r_ = (call);                                                                         \
        if (r_ != 0) return fail(RB_ERR_CUDA, std::string("NCCL: ") + (api)->GetErrorString(r_));      \
    } while (0)

extern "C" rb_status rb_comm_unique_id(rb_comm_id* id) {
    if (!id) return fail(RB_ERR_INVALID_ARGUMENT, "id is NULL");
    std::string why;
    NcclApi* api = nccl_api(&why);
    if (!api) return fail(RB_ERR_UNSUPPORTED, why);
    RB_NCCL(api->GetUniqueId(id), api);
    return RB_OK;
}

extern "C" rb_status rb_comm_init_rank(rb_context* ctx, int n_ranks, int rank, const rb_comm_id* id, rb_comm** out) {
    if (!ctx || !id || !out || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(RB_ERR_INVALID_ARGUMENT, "bad communicator arguments");
    std::string why;
    NcclApi* api = nccl_api(&why);
    if (!api) return fail(RB_ERR_UNSUPPORTED, why);
    RB_CUDA(cudaSetDevice(ctx->device));
    auto c = std::make_unique<rb_comm>();
    c->comms.resize(1), c->ctxs = {ctx}, c->n_ranks = n_ranks, c->rank = rank;
    RB_NCCL(api->CommInitRank(&c->comms[0], n_ranks, *id, rank), api);
    *out = c.release();
    return RB_OK;
}

extern "C" rb_status rb_comm_init_all(rb_context** ctxs, int n_gpus, rb_comm** out) {
    if (!ctxs || !out || n_gpus < 1) return fail(RB_ERR_INVALID_ARGUMENT, "bad communicator arguments");
    std::string why;
    NcclApi* api = nccl_api(&why);
    if (!api) return fail(RB_ERR_UNSUPPORTED, why);
    auto c = std::make_unique<rb_comm>();
    std::vector<int> devs(n_gpus);
    for (int i = 0; i < n_gpus; i++) {
        if (!ctxs[i]) return fail(RB_ERR_INVALID_ARGUMENT, "context is NULL");
        devs[i] = ctxs[i]->device, c->ctxs.push_back(ctxs[i]);
    }
    c->comms.resize(n_gpus), c->n_ranks = n_gpus;
    RB_NCCL(api->CommInitAll(c->comms.data(), n_gpus, devs.data()), api);
    *out = c.release();
    return RB_OK;
}

extern "C" rb_status rb_comm_destroy(rb_comm* c) {
    if (!c) return RB_OK;
    NcclApi* api = nccl_api(nullptr);
    for (rb_p2p* q : c->p2p) rb_p2p_destroy(q);
    if (api)
        for (void* k : c->comms)
            if (k) api->CommDestroy(k);
    delete c;
    return RB_OK;
}

// "p2p ..." or "nccl ...": how rb_batch_render_mix_allreduce exchanges the mixes on this communicator (known after the first call)
extern "C" rb_status rb_comm_transport(rb_comm* c, char* buf, uint64_t cap) {
    if (!c || !buf || cap == 0) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    snprintf(buf, (size_t)cap, "%s", c->transport.c_str());
    return RB_OK;
}

// Collective: every rank calls it with the same mix_len.  Leaves c->p2p empty (NCCL) when the ranks cannot map each other's memory.
static void comm_setup_p2p(rb_comm* c, NcclApi* api, uint64_t mix_len) {
    if (!c->p2p.empty() && rb_p2p_capacity(c->p2p[0]) >= mix_len) return;
    if (c->p2p_tried && c->p2p.empty()) return;                  // settled on NCCL
    c->p2p_tried = true;
    for (rb_p2p* q : c->p2p) rb_p2p_destroy(q);
    c->p2p.clear();
    const char* only = getenv("RB_COMM_NCCL_ONLY");
    if ((only && *only && *only != '0') || c->n_ranks < 2 || c->n_ranks > RB_P2P_MAX_RANKS) return;
    const uint64_t cap = std::max<uint64_t>(mix_len, 1ull << 16);
    std::string why;
    cudaError_t e;
    if (c->comms.size() == 1) {
        void* comm = c->comms[0];
        rb_p2p* p = nullptr;
        e = rb_p2p_create_rank(c->n_ranks, c->rank, c->ctxs[0]->device, c->ctxs[0]->stream, cap,
                               [api, comm](const void* s, void* r, size_t bytes, cudaStream_t st) {
                                   return api->AllGather(s, r, bytes, NCCL_INT8, comm, st) == 0 ? cudaSuccess : cudaErrorInvalidValue;
                               }, &p, &why);
        if (e == cudaSuccess && p) c->p2p = {p};
    } else {
        std::vector<int> devs;
        std::vector<cudaStream_t> sts;
        for (rb_context* x : c->ctxs) devs.push_back(x->device), sts.push_back(x->stream);
        std::vector<rb_p2p*> ps(c->ctxs.size(), nullptr);
        e = rb_p2p_create_local((int)ps.size(), devs.data(), sts.data(), cap, ps.data(), &why);
        if (e == cudaSuccess) c->p2p = ps;
    }
    if (!c->p2p.empty())
        c->transport = "p2p (k_mix_exchange: (value, tag) pairs pushed into every peer's mailbox over NVLink, summed in rank order)";
    else
        c->transport = "nccl (ncclAllReduce sum f32 on the render stream; peer memory not used: " + why + ")";
}

// Render every batch (one per local rank of the communicator, in rank order) and all-reduce the mixes in place: afterwards
// each rb_batch_mix_device_ptr holds the sum over ALL ranks.  Asynchronous on the contexts' streams like a render.
extern "C" rb_status rb_batch_render_mix_allreduce(rb_batch** batches, int n_local, rb_comm* c) {
    if (!batches || !c || n_local != (int)c->comms.size()) return fail(RB_ERR_INVALID_ARGUMENT, "one batch per local rank of the communicator");
    for (int i = 0; i < n_local; i++)
        if (batches[i] && batches[i]->has_master) return fail(RB_ERR_UNSUPPORTED, "a master chain runs on a single GPU's mix");
    NcclApi* api = nccl_api(nullptr);
    if (!api) return fail(RB_ERR_UNSUPPORTED, "NCCL is not loaded");
    for (int i = 0; i < n_local; i++) {
        if (!batches[i] || batches[i]->ctx != c->ctxs[i]) return fail(RB_ERR_INVALID_ARGUMENT, "batch i must live on the context of local rank i");
        if (batches[i]->mix_len != batches[0]->mix_len) return fail(RB_ERR_INVALID_ARGUMENT, "the shards must share the mixer timeline (equal mix_len)");
    }
    if (c->n_ranks > 1 && batches[0]->mix_len) comm_setup_p2p(c, api, batches[0]->mix_len);
    const bool p2p = !c->p2p.empty() && c->n_ranks > 1 && batches[0]->mix_len;
    for (int i = 0; i < n_local; i++) {
        const float* partial = nullptr;
        uint32_t n_rows = 0;
        uint64_t pstride = 0;
        const bool fuse = p2p && batches[i]->fused && !(batches[i]->flags & RB_KEEP_STREAM_OUTPUTS) &&
                          rb_fused_partial_rows(batches[i]->fused, &partial, &n_rows, &pstride);
        rb_status s = render_device(batches[i], fuse);
        if (s != RB_OK) return s;
        if (p2p) {   // ONE kernel: [the ordered sum of the shard's partial rows +] push to the peers + the rank-ordered sum
            RB_CUDA(cudaSetDevice(c->ctxs[i]->device));
            RB_CUDA(rb_p2p_allreduce(c->p2p[i], batches[i]->d_out, batches[i]->mix_len, fuse ? partial : nullptr, n_rows, pstride, c->ctxs[i]->stream));
        }
    }
    if (c->n_ranks == 1 || batches[0]->mix_len == 0 || p2p) return RB_OK;
    if (n_local > 1) RB_NCCL(api->GroupStart(), api);
    for (int i = 0; i < n_local; i++) {
        RB_CUDA(cudaSetDevice(c->ctxs[i]->device));
        RB_NCCL(api->AllReduce(batches[i]->d_out, batches[i]->d_out, (size_t)batches[i]->mix_len, NCCL_FLOAT32, NCCL_SUM, c->comms[i], c->ctxs[i]->stream), api);
    }
    if (n_local > 1) RB_NCCL(api->GroupEnd(), api);
    return RB_OK;
}

extern "C" rb_status rb_batch_mix_device_ptr(rb_batch* b, float** dptr) {
    if (!b || !dptr) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *dptr = b->d_out;
    return RB_OK;
}
extern "C" rb_status rb_batch_render_mix(rb_batch* b, float* out_host, uint64_t max_samples, uint64_t* written) {
    rb_status s = rb_batch_render_mix_device(b);
    if (s != RB_OK) return s;
    uint64_t n = std::min<uint64_t>(b->mix_len, max_samples);
    if (n && !out_host) return fail(RB_ERR_INVALID_ARGUMENT, "out_host is NULL");
    if (n) RB_CUDA(cudaMemcpyAsync(out_host, b->d_out, n * 4, cudaMemcpyDeviceToHost, b->ctx->stream));
    RB_CUDA(cudaStreamSynchronize(b->ctx->stream));
    if (written) *written = n;
    return RB_OK;
}
extern "C" rb_status rb_batch_read_mix(rb_batch* b, uint64_t offset, float* out_host, uint64_t n_samples, uint64_t* written) {
    if (!b) return fail(RB_ERR_INVALID_ARGUMENT, "batch is NULL");
    if (!b->rendered) return fail(RB_ERR_STATE, "render first");
    uint64_t n = offset >= b->mix_len ? 0 : std::min<uint64_t>(n_samples, b->mix_len - offset);
    if (n && !out_host) return fail(RB_ERR_INVALID_ARGUMENT, "out_host is NULL");
    RB_CUDA(cudaSetDevice(b->ctx->device));
    if (n) RB_CUDA(cudaMemcpyAsync(out_host, b->d_out + offset, n * 4, cudaMemcpyDeviceToHost, b->ctx->stream));
    RB_CUDA(cudaStreamSynchronize(b->ctx->stream));
    if (written) *written = n;
    return RB_OK;
}
extern "C" rb_status rb_batch_read_stream(rb_batch* b, size_t stream, float* out_host, uint64_t max_samples,
                                          uint64_t* written) {
    rb_status s = check_stream(b, stream);
    if (s != RB_OK) return s;
    if (!b->rendered) return fail(RB_ERR_STATE, "render first");
    PlanStream& ps = b->streams[stream];
    if (!ps.final_ptr) return fail(RB_ERR_STATE, "per-stream outputs need RB_KEEP_STREAM_OUTPUTS on a fused batch");
    if (ps.nodes.empty() && ps.desc.format != RB_FMT_F32) return fail(RB_ERR_STATE, "internal: unconverted stream");
    uint64_t n = std::min<uint64_t>(ps.out_len, max_samples);
    if (n && !out_host) return fail(RB_ERR_INVALID_ARGUMENT, "out_host is NULL");
    RB_CUDA(cudaSetDevice(b->ctx->device));
    if (n) RB_CUDA(cudaMemcpyAsync(out_host, ps.final_ptr, n * 4, cudaMemcpyDeviceToHost, b->ctx->stream));
    RB_CUDA(cudaStreamSynchronize(b->ctx->stream));
    if (written) *written = n;
    return RB_OK;
}

// ------------------------------------------------------------------------------------------------
// stand-alone conversions (SampleRateConverter / ChannelCountConverter / SampleTypeConverter)
// ------------------------------------------------------------------------------------------------
extern "C" rb_status rb_sample_rate_out_len(uint64_t n_in, uint32_t from, uint32_t to, uint16_t ch, uint64_t* n_out) {
    if (!n_out) return fail(RB_ERR_INVALID_ARGUMENT, "n_out is NULL");
    if (from == 0 || to == 0 || ch == 0) return fail(RB_ERR_INVALID_ARGUMENT, "zero rate or channels (rodio panics)");
    if (n_in % ch) return fail(RB_ERR_UNALIGNED_FRAMES, "n_in % channels != 0");
    uint32_t g = std::gcd(from, to);
    uint32_t f = from / g, t = to / g;
    if (f != t && (uint64_t)f * t >= (1ull << 32)) return fail(RB_ERR_RATIO_OVERFLOW, "reduced from*to >= 2^32");
    *n_out = src_out_frames(n_in / ch, f, t) * ch;
    return RB_OK;
}
extern "C" rb_status rb_channels_out_len(uint64_t n_in, uint16_t from, uint16_t to, uint64_t* n_out) {
    if (!n_out) return fail(RB_ERR_INVALID_ARGUMENT, "n_out is NULL");
    if (from == 0 || to == 0) return fail(RB_ERR_INVALID_ARGUMENT, "zero channels (rodio panics)");
    if (n_in % from) return fail(RB_ERR_UNALIGNED_FRAMES, "n_in % from != 0");
    *n_out = n_in / from * to;
    return RB_OK;
}

static rb_status run_single_uniform(rb_context* ctx, const float* in, uint64_t n_in, uint32_t c_in, uint32_t rate_in,
                                    uint32_t c_out, uint32_t rate_out, float* out, uint64_t cap, uint64_t* n_out) {
    if (!ctx || (!in && n_in) || !n_out) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (c_in > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "more than 12 channels");
    PlanNode nd;
    rb_status s = plan_uniform(nd, n_in, c_in, rate_in, 0, c_out, rate_out);
    if (s != RB_OK) return s;
    *n_out = nd.d.n_out;
    if (nd.d.n_out > cap) return fail(RB_ERR_BUFFER_TOO_SMALL, "output capacity too small");
    if (nd.d.n_out == 0) return RB_OK;
    if (!out) return fail(RB_ERR_INVALID_ARGUMENT, "out is NULL");
    RB_CUDA(cudaSetDevice(ctx->device));
    float *d_in = nullptr, *d_out = nullptr;
    rb_node_dev* d_node = nullptr;
    RB_CUDA(cudaMalloc(&d_in, n_in * 4 + 16));
    RB_CUDA(cudaMalloc(&d_out, nd.d.n_out * 4));
    RB_CUDA(cudaMalloc(&d_node, sizeof(rb_node_dev)));
    nd.d.src = d_in, nd.d.dst = d_out;
    cudaError_t e = cudaMemcpyAsync(d_in, in, n_in * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_node, &nd.d, sizeof(rb_node_dev), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = rb_launch_nodes(RB_N_UNIFORM, d_node, 1, nd.d.n_out, c_in, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, nd.d.n_out * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d_in), cudaFree(d_out), cudaFree(d_node);
    if (e != cudaSuccess) return fail(RB_ERR_CUDA, cudaGetErrorString(e));
    return RB_OK;
}

extern "C" rb_status rb_convert_sample_rate(rb_context* ctx, const float* in, uint64_t n_in, uint32_t from, uint32_t to,
                                            uint16_t channels, float* out, uint64_t cap, uint64_t* n_out) {
    if (from == 0 || to == 0 || channels == 0) return fail(RB_ERR_INVALID_ARGUMENT, "zero rate or channels (rodio panics)");
    if (n_in % channels) return fail(RB_ERR_UNALIGNED_FRAMES, "n_in % channels != 0");
    return run_single_uniform(ctx, in, n_in, channels, from, channels, to, out, cap, n_out);
}
extern "C" rb_status rb_convert_channels(rb_context* ctx, const float* in, uint64_t n_in, uint16_t from, uint16_t to,
                                         float* out, uint64_t cap, uint64_t* n_out) {
    if (from == 0 || to == 0) return fail(RB_ERR_INVALID_ARGUMENT, "zero channels (rodio panics)");
    if (n_in % from) return fail(RB_ERR_UNALIGNED_FRAMES, "n_in % from != 0");
    if (from == to) {   // ChannelCountConverter with from == to is the identity map
        if (!n_out) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
        *n_out = n_in;
        if (n_in > cap) return fail(RB_ERR_BUFFER_TOO_SMALL, "output capacity too small");
        if (n_in) memcpy(out, in, n_in * 4);
        return RB_OK;
    }
    return run_single_uniform(ctx, in, n_in, from, 48000, to, 48000, out, cap, n_out);
}
extern "C" rb_status rb_convert_samples(rb_context* ctx, const void* in, rb_sample_format in_fmt, void* out,
                                        rb_sample_format out_fmt, uint64_t n) {
    if (!ctx || ((!in || !out) && n)) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    if ((uint32_t)in_fmt > RB_FMT_I24_IN_I32 || (uint32_t)out_fmt > RB_FMT_I24_IN_I32)
        return fail(RB_ERR_INVALID_ARGUMENT, "unknown sample format");
    if (in_fmt != RB_FMT_F32 && out_fmt != RB_FMT_F32)
        return fail(RB_ERR_UNSUPPORTED, "one side of the conversion must be f32 (the Source sample type)");
    if (n == 0) return RB_OK;
    RB_CUDA(cudaSetDevice(ctx->device));
    void *d_in = nullptr, *d_out = nullptr;
    RB_CUDA(cudaMalloc(&d_in, n * fmt_size(in_fmt)));
    RB_CUDA(cudaMalloc(&d_out, n * fmt_size(out_fmt)));
    cudaError_t e = cudaMemcpyAsync(d_in, in, n * fmt_size(in_fmt), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = rb_launch_convert(d_in, in_fmt, d_out, out_fmt, n, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, n * fmt_size(out_fmt), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d_in), cudaFree(d_out);
    if (e != cudaSuccess) return fail(RB_ERR_CUDA, cudaGetErrorString(e));
    return RB_OK;
}


// ------------------------------------------------------------------------------------------------
// streaming sessions (block form of MixerSource::next for sources that arrive incrementally)
// ------------------------------------------------------------------------------------------------
// Bookkeeping: rb_session_plan.h (plain host code, also run by the CPU emulator of tests/emu/);
// kernel: k_fused_lanes over per-block rows (rb_lanes_core.h: o0 / i0 / state / ROW_CONTINUES).
// Slot rows: the lane kernel carries at most two channels per lane (CI == CO, or CI = 1 and CO = 2), so a source is served by
// one row per pair of the mixer channels it feeds (rb_lanes.h, rb_fifo_job).  Output channel j of ChannelCountConverter
// (src/conversions/channels.rs:57-85) is input channel j if j < CI, channel 0 again if j == 1 and CI == 1, else 0.0: the rows
// cover every channel of the first kind and of the second; a channel of the third kind gets no row, because +-0 added to a
// sum that starts from +0.0 changes nothing -- as long as the filter and the gain behind the conversion are finite
// (rb_session_create refuses the other sources).
struct rb_session {
    rb_context* ctx = nullptr;
    uint32_t mixer_rate = 0;
    uint32_t channels = 1;        // of the mixer (1 .. RB_MAX_CHANNELS)
    std::vector<uint8_t> src_ch;  // per source (source order): its own channel count
    std::vector<uint8_t> pads;    // per source: its conversion pads channels with 0.0 (1), its take pads its last frame (2)
    bool has_biquad = false, has_post = false;
    // Sources may have different rates (each at or below the mixer's): one kernel launch per reduced rate pair.  All
    // per-source arrays below are in SOURCE ORDER (stable partition by rate pair, channels and chain variant); pos[] maps the
    // caller's index to it.
    std::vector<uint32_t> pos;
    std::vector<session::Stream> st;
    std::vector<float> coef;      // 5 per stream
    std::vector<float> ffk, post, pre, mid;
    std::vector<float> vol_a, vol_b;   // the factor the two frames in front of Stream::fpos were pulled with (rb_session_set_volume)
    // Rows are in CLASS ORDER: the rows of the sources in the caller's order, each source's slots in channel order, stably
    // partitioned by (rate pair, chain variant, slot).  One launch per class; k_sum_slots adds the partial rows in that order.
    // FIFOs, filter states and input flags are per row; positions, gains and the queue are per source.
    struct Slot {
        uint32_t src;             // source order
        uint8_t ch0, w, ci;       // mixer channels [ch0, ch0 + w), fed by source channels [ch0, ch0 + ci) (ci = 1, w = 2: mono repeated)
    };
    struct Class {
        uint32_t first = 0, count = 0, ch_in = 1, ch_out = 1;
        bool has_biquad = false, ff2 = false, has_pre = false, front = false;
    };
    std::vector<Class> classes;
    std::vector<Slot> rows;
    std::vector<std::vector<uint32_t>> rows_of;   // per source: its rows, in slot order
    bool plain = true;            // every source is one row that carries all of its channels: the version-5 state blob
    uint32_t n_groups = 0;        // partial rows: one per warp, every class rounds up on its own
    uint64_t T = 0;               // mixer frames rendered so far
    uint32_t fifo_cap = 0, max_block = 0, max_src_ch = 1;
    uint64_t stride = 0;          // floats per row in a FIFO arena
    float* d_fifo[2] = {nullptr, nullptr};
    int cur = 0;
    float *d_state = nullptr, *d_zeros = nullptr, *d_partial = nullptr, *d_out = nullptr;   // d_state: 8 floats per row
    uint32_t* d_flags = nullptr;  // per row, sticky: a pushed frame was outside the exact-reciprocal class
    lanes::Row* d_rows = nullptr;
    uint32_t* d_u32 = nullptr;    // [2][rows]: drop, keep (render)
    uint32_t* d_slot = nullptr;   // per partial row: ch0 | w << 16 (k_sum_slots)
    rb_fifo_job* d_jobs = nullptr;   // [rows]: the scatter of one push
    float* d_stage = nullptr;     // push staging, [n * fifo_cap * max_src_ch], allocated by the first push
    // pinned host mirrors, reused by every call (each call ends with a stream synchronisation)
    lanes::Row* h_rows = nullptr;
    uint32_t* h_u32 = nullptr;
    rb_fifo_job* h_jobs = nullptr;
    float* h_out = nullptr;
    // adapters on the MixerSource (rb_session_set_master).  The limiter state is double-buffered: a block reads
    // d_master[master_k] and writes d_master[master_k ^ 1]; master_k flips once the block's synchronisation succeeded.
    bool has_master = false;
    rb_master_params master{};
    float* d_master[2] = {nullptr, nullptr};   // integ[C], peak[C]
    int master_k = 0;
    rb_master_run* d_master_runs = nullptr;    // the block's active runs, [n_streams]
    rb_master_run* h_master_runs = nullptr;
    // push programs (rb_lanes.h: rb_prog_op): the closed-form adapters a source's chain begins with, applied by the scatter of
    // every push.  Per source (source order): its ops, the frames that went through them, and where its take ends the source.
    bool has_prog = false;
    std::vector<rb_prog_op> prog_ops;
    std::vector<uint32_t> prog_op0, prog_n;
    std::vector<uint64_t> prog_pos;
    std::vector<uint64_t> prog_end;            // frames: the take's count padded to whole frames; ~0: no take
    std::vector<uint8_t> no_silence;           // a take in front of a resampling conversion: rb_session_push_silence refused
    rb_prog_op* d_prog = nullptr;
    rb_fifo_prog_job *d_pjobs = nullptr, *h_pjobs = nullptr;
    // restart schedules (RB_SESSION_RESTARTS, rb_session_plan.h): some source has one; the cuts of a block, rows in compressed
    // sparse row form (cut_first: [rows + 1]), grown to the largest block's count
    bool restarts = false, has_sched = false;
    lanes::Cut *d_cuts = nullptr, *h_cuts = nullptr;
    uint32_t *d_cut_first = nullptr, *h_cut_first = nullptr;
    size_t cut_cap = 0;
    uint64_t restart_launches = 0;             // launches of the lane kernel's RESTART twins so far
    // span marks (rb_session_push_spans): per source, what current_span_len() reports at the pushed end (samples, 0: None) --
    // desc.span_len until a mark says otherwise -- and the run cap a report of None gives (a take's, or none); `marked`: some push
    // carried marks (the state blob is version 9 from then on)
    std::vector<uint64_t> report, none_cap;
    std::vector<uint8_t> follows_marks;        // the source is resampled in a session with RB_SESSION_RESTARTS: marks move its runs
    bool marked = false;
    // generator sources (RB_FX_SIGNAL): the session generates their samples into their FIFOs before each render, as if they had been
    // pushed.  Per source (source order) its phase slot (~0u: not a generator); per slot the source, the function, the phase step
    // and the samples `.take(n)` lets through (~0: endless).  The phase of every generator's next sample lives on the device,
    // double-buffered like the limiter state: a fill reads d_phase[phase_k] and writes d_phase[phase_k ^ 1], and phase_k flips once
    // the render's synchronisation succeeded.  gen_frames: the samples the fill of the current render writes.
    std::vector<uint32_t> gen_of, gens, gen_fn;
    std::vector<float> gen_step;
    std::vector<uint64_t> gen_end;
    float* d_phase[2] = {nullptr, nullptr};
    int phase_k = 0;
    uint64_t gen_frames = 0;
    rb_fifo_gen_job *d_gjobs = nullptr, *h_gjobs = nullptr;
#if defined(RB_SIMT_EMULATE)
    std::vector<uint64_t> emu_fast_tiles;      // CPU build: fast tiles the emulator ran per class (rb_session_emu_fast_tiles)
#endif
};

extern "C" rb_status rb_session_destroy(rb_session* s) {
    if (!s) return RB_OK;
    if (s->ctx) cudaSetDevice(s->ctx->device);
    cudaFree(s->d_fifo[0]), cudaFree(s->d_fifo[1]), cudaFree(s->d_state), cudaFree(s->d_zeros), cudaFree(s->d_partial);
    cudaFree(s->d_out), cudaFree(s->d_flags), cudaFree(s->d_rows), cudaFree(s->d_u32), cudaFree(s->d_slot), cudaFree(s->d_jobs), cudaFree(s->d_stage);
    cudaFreeHost(s->h_rows), cudaFreeHost(s->h_u32), cudaFreeHost(s->h_jobs), cudaFreeHost(s->h_out);
    cudaFree(s->d_master[0]), cudaFree(s->d_master[1]), cudaFree(s->d_master_runs), cudaFreeHost(s->h_master_runs);
    cudaFree(s->d_prog), cudaFree(s->d_pjobs), cudaFreeHost(s->h_pjobs);
    cudaFree(s->d_cuts), cudaFreeHost(s->h_cuts), cudaFree(s->d_cut_first), cudaFreeHost(s->h_cut_first);
    cudaFree(s->d_phase[0]), cudaFree(s->d_phase[1]), cudaFree(s->d_gjobs), cudaFreeHost(s->h_gjobs);
    delete s;
    return RB_OK;
}

extern "C" rb_status rb_session_create(rb_context* ctx, uint16_t mixer_channels, uint32_t mixer_rate, const rb_stream_desc* descs,
                                       size_t n_streams, uint32_t fifo_frames, uint32_t max_block_frames, rb_session** out) {
    return rb_session_create_ex(ctx, mixer_channels, mixer_rate, descs, n_streams, fifo_frames, max_block_frames, 0, out);
}

extern "C" rb_status rb_session_create_ex(rb_context* ctx, uint16_t mixer_channels, uint32_t mixer_rate, const rb_stream_desc* descs,
                                          size_t n_streams, uint32_t fifo_frames, uint32_t max_block_frames, uint32_t flags, rb_session** out) {
    if (!ctx || !out || !descs) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (flags & ~(uint32_t)RB_SESSION_RESTARTS) return fail(RB_ERR_INVALID_ARGUMENT, "unknown session flags");
    const bool restarts = (flags & RB_SESSION_RESTARTS) != 0;
    if (mixer_rate == 0 || mixer_channels == 0 || n_streams == 0 || n_streams > 0x7FFFFFFFull)
        return fail(RB_ERR_INVALID_ARGUMENT, "zero mixer rate / channels or no streams");
    if (mixer_channels > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, "mixer: more than 12 channels");
    if (fifo_frames < 64 || max_block_frames == 0) return fail(RB_ERR_INVALID_ARGUMENT, "fifo_frames < 64 or max_block_frames == 0");
    if ((uint64_t)fifo_frames * RB_MAX_CHANNELS >= (1ull << 32))   // per-stream float counts travel as 32-bit words
        return fail(RB_ERR_OUT_OF_MEMORY, "fifo_frames too large (fifo_frames * channels must stay below 2^32)");
    std::unique_ptr<rb_session, rb_status (*)(rb_session*)> s(new (std::nothrow) rb_session, rb_session_destroy);
    if (!s) return fail(RB_ERR_OUT_OF_MEMORY, "host allocation failed");
    s->ctx = ctx, s->mixer_rate = mixer_rate, s->channels = mixer_channels, s->fifo_cap = fifo_frames, s->max_block = max_block_frames;
    const size_t n = n_streams;
    // pass 1: validate, find every source's reduced rate pair -> classes
    std::vector<uint32_t> from(n), to(n), chs(n), first_fx(n), key(n);
    std::vector<float> pre_of(n, 1.0f), mid_of(n, 1.0f);
    std::vector<uint32_t> front_fx(n, 0xFFFFFFFFu), front_rate(n, 0);
    std::vector<std::vector<rb_prog_op>> progs(n);
    std::vector<uint64_t> take_n(n, ~0ull);   // samples the source's takes let through
    std::vector<uint8_t> no_silence(n, 0);
    std::vector<uint64_t> run_cap(n, 0);      // RB_SESSION_RESTARTS: frames per converter run (0: the source is one run)
    std::vector<uint64_t> none_cap(n, session::NO_LIMIT);   // ... under a report of None
    std::vector<float> gen_step(n, 0.0f);     // generator sources: their phase step (gen[i])
    std::vector<uint8_t> gen(n, 0);
    for (size_t i = 0; i < n; i++) {
        const rb_stream_desc& d = descs[i];
        const std::string where = "stream " + std::to_string(i) + ": ";
        if (d.sample_rate == 0 || d.channels == 0) return fail(RB_ERR_INVALID_ARGUMENT, where + "zero sample rate or channels");
        if (d.n_effects && !d.effects) return fail(RB_ERR_INVALID_ARGUMENT, where + "effects is NULL");
        for (uint32_t k = 1; k < d.n_effects; k++)
            if (d.effects[k].kind == RB_FX_SIGNAL)
                return fail(RB_ERR_INVALID_ARGUMENT, where + "signal generator: only as effects[0] of an empty mono f32 span-less descriptor");
        gen[i] = d.n_effects && d.effects[0].kind == RB_FX_SIGNAL;
        if (gen[i]) {   // SignalGenerator::with_function (signal_generator.rs:107-128), validated as plan_stream does
            const rb_effect& e = d.effects[0];
            if (d.n_samples != 0 || d.channels != 1 || d.format != RB_FMT_F32 || d.span_len != 0)
                return fail(RB_ERR_INVALID_ARGUMENT, where + "signal generator: only as effects[0] of an empty mono f32 span-less descriptor");
            if (e.u32[0] > RB_SIGNAL_SAWTOOTH) return fail(RB_ERR_INVALID_ARGUMENT, where + "signal generator: unknown function");
            if (!(e.f32[0] > 0.0f)) return fail(RB_ERR_INVALID_ARGUMENT, where + "signal generator: frequency must be greater than zero");
            if (!std::isfinite(e.f32[0])) return fail(RB_ERR_UNSUPPORTED, where + "signal generator: infinite frequency");
            volatile float period = (float)d.sample_rate / e.f32[0];     // :118, the expression plan_stream uses
            gen_step[i] = 1.0f / period;                                 // :119
        }
        if (d.format != RB_FMT_F32) return fail(RB_ERR_UNSUPPORTED, where + "sessions take f32 sources");
        if (d.channels > RB_MAX_CHANNELS) return fail(RB_ERR_UNSUPPORTED, where + "more than 12 channels");
        if (mixer_channels == 1 && d.channels != 1) return fail(RB_ERR_UNSUPPORTED, where + "a mono mixer takes mono sources");
        chs[i] = d.channels;
        // The push program: effects [0, p), p one past the last LINEAR_RAMP / TAKE_DURATION / DISTORTION in front of everything
        // else.  No state depends on the signal there: every output sample is a function of its input sample and its index in
        // the source, so the scatter of each push applies them.  Each one sees the rate the SPEEDs in front of it report.
        // A generator is the source itself: what follows it is a chain as for pushed PCM.
        const uint32_t k_src = gen[i] ? 1u : 0u;
        uint32_t p = k_src, rate = d.sample_rate;
        for (uint32_t k = k_src; k < d.n_effects; k++) {
            const uint32_t kd = d.effects[k].kind;
            if (kd == RB_FX_LINEAR_RAMP || kd == RB_FX_TAKE_DURATION || kd == RB_FX_DISTORTION) p = k + 1;
            else if (kd != RB_FX_AMPLIFY && kd != RB_FX_SPEED) break;
        }
        bool take_open = false;   // ops behind a take that ends inside a frame see its 0.0 padding
        for (uint32_t k = k_src; k < p; k++) {
            const rb_effect& e = d.effects[k];
            if (e.kind == RB_FX_SPEED) {
                rate = rb_speed_sample_rate(rate, e.f32[0]);
                if (rate == 0) return fail(RB_ERR_INVALID_ARGUMENT, where + "speed: zero sample rate");
                continue;
            }
            rb_prog_op op;
            memset(&op, 0, sizeof(op));
            if (e.kind == RB_FX_AMPLIFY) {
                op.kind = RB_N_AMPLIFY, op.p.amp = e.f32[0];
            } else {
                rb_node_dev nd;
                memset(&nd, 0, sizeof(nd));
                rb_status st = plan_pointwise(e, rate, d.channels, nd);
                if (st != RB_OK) return st;
                if (nd.kind == RB_N_TAKE) {
                    if (nd.p.take.dps_ns == 0) return fail(RB_ERR_INVALID_ARGUMENT, where + "take_duration: the duration per sample is 0");
                    take_n[i] = std::min(take_n[i], nd.p.take.count);
                }
                op.kind = nd.kind;
                memcpy(&op.p, &nd.p, sizeof(op.p));
            }
            // the padding is 0.0: every factor behind it keeps it a zero, as rodio never pulls it (it only completes the frame)
            if (take_open && !(op.kind == RB_N_AMPLIFY ? std::isfinite(op.p.amp)
                               : op.kind == RB_N_DISTORT ? std::isfinite(op.p.dist.gain)
                               : op.kind == RB_N_RAMP ? std::isfinite(op.p.ramp.start) && std::isfinite(op.p.ramp.end) : true))
                return fail(RB_ERR_UNSUPPORTED, where + "a non-finite factor behind a take that ends inside a frame (rodio never pulls its padding)");
            if (op.kind == RB_N_TAKE && op.p.take.count % d.channels) take_open = true;
            progs[i].push_back(op);
        }
        // Source::speed in front of the conversion only changes the rate the source reports (src/source/speed.rs:130-133);
        // one Source::amplify there -- `source.amplify(v)` handed to Mixer::add -- scales every frame before it is interpolated
        // (src/source/amplify.rs:91-95).  The two commute: one touches the samples, the other the reported rate.
        uint32_t k0 = p;
        bool has_pre = false, has_mid = false, front = false;
        // A filter there as well -- `source.low_pass(f)` handed to the mixer, or appended to a Player, which keeps its volume
        // behind it (src/player.rs:120-128) -- runs at the rate its input reports at that point (src/source/blt.rs:
        // to_applier(input.sample_rate())), once per input frame; one gain in front of it, one behind.
        while (k0 < d.n_effects) {
            const rb_effect& e = d.effects[k0];
            if (e.kind == RB_FX_SPEED) rate = rb_speed_sample_rate(rate, e.f32[0]);
            else if (e.kind == RB_FX_AMPLIFY && !front && !has_pre) has_pre = true, pre_of[i] = e.f32[0];
            else if (e.kind == RB_FX_AMPLIFY && front && !has_mid) has_mid = true, mid_of[i] = e.f32[0];
            else if ((e.kind == RB_FX_LOW_PASS || e.kind == RB_FX_HIGH_PASS) && !front) front = true, front_fx[i] = k0, front_rate[i] = rate;
            else break;
            k0++;
        }
        first_fx[i] = k0;
        if (k0 >= d.n_effects || d.effects[k0].kind != RB_FX_UNIFORM || d.effects[k0].u32[0] != mixer_channels || d.effects[k0].u32[1] != mixer_rate)
            return fail(RB_ERR_UNSUPPORTED, where + "the chain must be [SPEED | AMPLIFY | one filter] UNIFORM(mixer channels, mixer rate) ...");
        const uint32_t g = std::gcd(rate, mixer_rate);
        from[i] = rate / g, to[i] = mixer_rate / g;
        const bool filtered = k0 + 1 < d.n_effects && (d.effects[k0 + 1].kind == RB_FX_LOW_PASS || d.effects[k0 + 1].kind == RB_FX_HIGH_PASS);
        if (front && filtered) return fail(RB_ERR_UNSUPPORTED, where + "one filter per source: in front of the conversion or behind it");
        // With RB_SESSION_RESTARTS the mixer's conversion is restarted where rodio restarts it: every min(span_len, 32768) samples,
        // behind a take every min(samples left in the take, 32768).  Served when every run is whole frames of the source.
        const bool cap_whole = RB_UNIFORM_SPAN_CAP % d.channels == 0;
        bool take_runs = false;   // a resampled take that the schedule follows
        if (restarts) {
            if (d.span_len % d.channels || (d.span_len > RB_UNIFORM_SPAN_CAP && !cap_whole))
                return fail(RB_ERR_UNSUPPORTED, where + "restarts: span_len (capped at 32768 samples) must be whole frames of the source");
            take_runs = from[i] != to[i] && take_n[i] != ~0ull && take_n[i] % d.channels == 0 && (take_n[i] <= RB_UNIFORM_SPAN_CAP || cap_whole);
            if (take_runs) none_cap[i] = cap_whole ? RB_UNIFORM_SPAN_CAP / d.channels : take_n[i] / d.channels;
            if (from[i] != to[i] && (d.span_len || take_runs)) {
                run_cap[i] = d.span_len ? std::min(d.span_len, RB_UNIFORM_SPAN_CAP) / d.channels : none_cap[i];
                if (run_cap[i] < 2) return fail(RB_ERR_UNSUPPORTED, where + "restarts: converter runs shorter than two frames");
            }
        }
        if (take_n[i] != ~0ull) {
            // Behind a take the mixer's conversion re-bootstraps every min(samples left, 32768) samples (src/source/uniform.rs:50-68,
            // take.rs:180-196) and never pulls the padding of the take's last frame.  A session converts the source as one run, with
            // the padding: the same samples when the take is one run of whole frames, or when the conversion keeps no state across a
            // restart -- the source's own rate, and channels passed through or restarted on a frame boundary.
            const uint64_t C_in = d.channels;
            const bool whole = take_n[i] % C_in == 0;
            const bool one_run = whole && take_n[i] <= RB_UNIFORM_SPAN_CAP;
            const bool stateless = from[i] == to[i] && (take_n[i] <= RB_UNIFORM_SPAN_CAP || C_in == 1 || C_in == mixer_channels || RB_UNIFORM_SPAN_CAP % C_in == 0);
            if (!one_run && !stateless && !take_runs)
                return fail(RB_ERR_UNSUPPORTED, where + "take_duration: the mixer's conversion restarts every 32768 samples behind a take; "
                                                        "sessions serve longer takes (or takes that end inside a frame) at the mixer's rate only");
            if (!whole && (front || filtered))
                return fail(RB_ERR_UNSUPPORTED, where + "a take that ends inside a frame pads it with 0.0, which a filter would see (rodio never pulls it)");
            // Pausable passes the take's span on: the conversion then counts the pause's zeros against the take and restarts early
            if (from[i] != to[i] && !take_runs) no_silence[i] = 1;
        }
        // filtered / unfiltered sources, sources with / without a gain in front and sources whose filter sits in front are
        // classes of their own (a filter in front always applies the gains around it: no class of its own for those)
        key[i] = d.channels | (filtered ? 0x100u : 0u) | (has_pre && !front ? 0x200u : 0u) | (front ? 0x400u : 0u);
        if (from[i] > (1u << 20) || to[i] > (1u << 20))
            return fail(RB_ERR_RATIO_OVERFLOW, where + "reduced rate pair beyond 2^20");
    }
    s->pos.assign(n, 0);
    std::vector<uint32_t> order;   // source order -> caller's index
    for (const auto& cls : lanes::classes_by_ratio(from.data(), to.data(), key.data(), (uint32_t)n))
        for (uint32_t i : cls) s->pos[i] = (uint32_t)order.size(), order.push_back(i);
    // pass 2: chains, in source order
    s->st.resize(n), s->coef.assign(5 * n, 0.0f), s->ffk.assign(n, 0.0f), s->post.assign(n, 1.0f), s->pre.assign(n, 1.0f), s->mid.assign(n, 1.0f), s->src_ch.assign(n, 1);
    s->vol_a.assign(n, 1.0f), s->vol_b.assign(n, 1.0f), s->pads.assign(n, 0);
    s->prog_op0.assign(n, 0), s->prog_n.assign(n, 0), s->prog_pos.assign(n, 0), s->prog_end.assign(n, ~0ull), s->no_silence.assign(n, 0);
    s->restarts = restarts, s->report.assign(n, 0), s->none_cap.assign(n, session::NO_LIMIT), s->follows_marks.assign(n, 0);
    s->gen_of.assign(n, ~0u);
    bool any_biquad = false;
    std::vector<uint8_t> row_ff2(n, 1);
    for (size_t r = 0; r < n; r++) {
        const size_t i = order[r];
        const rb_stream_desc& d = descs[i];
        const std::string where = "stream " + std::to_string(i) + ": ";
        uint32_t k = first_fx[i] + 1;   // behind [SPEED | AMPLIFY] UNIFORM
        s->pre[r] = pre_of[i], s->mid[r] = mid_of[i];
        s->vol_a[r] = s->vol_b[r] = front_fx[i] != 0xFFFFFFFFu ? mid_of[i] : pre_of[i];
        bool biq = false;
        if (front_fx[i] != 0xFFFFFFFFu) {
            const rb_effect& e = d.effects[front_fx[i]];
            if (e.u32[0] == 0 || !(e.f32[0] > 0.0f)) return fail(RB_ERR_INVALID_ARGUMENT, where + "filter frequency and q must be positive");
            const hostmath::Blt c = hostmath::blt(e.kind == RB_FX_HIGH_PASS, e.u32[0], e.f32[0], front_rate[i]);
            float* co = &s->coef[5 * r];
            co[0] = c.b0, co[1] = c.b1, co[2] = c.b2, co[3] = c.a1, co[4] = c.a2;
            row_ff2[r] = 0, biq = true;
            s->st[r].front = true;
        }
        bool behind = false;   // a filter behind the conversion: it also filters the channels the conversion pads
        if (k < d.n_effects && (d.effects[k].kind == RB_FX_LOW_PASS || d.effects[k].kind == RB_FX_HIGH_PASS)) {
            const rb_effect& e = d.effects[k];
            if (e.u32[0] == 0 || !(e.f32[0] > 0.0f)) return fail(RB_ERR_INVALID_ARGUMENT, where + "filter frequency and q must be positive");
            const hostmath::Blt c = hostmath::blt(e.kind == RB_FX_HIGH_PASS, e.u32[0], e.f32[0], mixer_rate);
            float* co = &s->coef[5 * r];
            co[0] = c.b0, co[1] = c.b1, co[2] = c.b2, co[3] = c.a1, co[4] = c.a2;
            if (!lanes::ff2_coeffs(c.b0, c.b1, c.b2, &s->ffk[r])) row_ff2[r] = 0;
            biq = behind = true, k++;
        }
        any_biquad |= biq;
        if (k < d.n_effects && d.effects[k].kind == RB_FX_AMPLIFY) s->post[r] = d.effects[k].f32[0], s->has_post = true, k++;
        if (k != d.n_effects) return fail(RB_ERR_UNSUPPORTED, where + "chain shape: [SPEED | AMPLIFY | one filter] UNIFORM [LOW_PASS | HIGH_PASS] [AMPLIFY]");
        // Channels the conversion pads get no row: their 0.0 must stay a zero behind the filter and the gain
        s->pads[r] = mixer_channels > (d.channels == 1 ? 2u : d.channels);
        if (take_n[i] != ~0ull && take_n[i] % d.channels) {   // ... and so must the padding of a take's last frame, behind every gain
            s->pads[r] |= 2;
            if (!std::isfinite(pre_of[i]) || !std::isfinite(mid_of[i]))
                return fail(RB_ERR_UNSUPPORTED, where + "a take that ends inside a frame, behind a non-finite gain (rodio never pulls its padding)");
        }
        if (s->pads[r]) {
            const float* co = &s->coef[5 * r];
            bool finite = std::isfinite(s->post[r]);
            for (int j = 0; j < 5 && behind; j++) finite = finite && std::isfinite(co[j]);
            if (!finite)
                return fail(RB_ERR_UNSUPPORTED, where + "the conversion pads channels with 0.0 and the filter or gain behind it is not finite (rodio gives NaN there)");
        }
        s->st[r].mix_start = d.mix_start, s->st[r].from = from[i], s->st[r].to = to[i];
        s->st[r].run_cap = run_cap[i], s->has_sched = s->has_sched || run_cap[i] != 0;
        s->report[r] = d.span_len, s->none_cap[r] = none_cap[i], s->follows_marks[r] = restarts && from[i] != to[i];
        if (d.mix_start == RB_SESSION_HELD) s->st[r].held = true, s->st[r].mix_start = 0;   // Mixer::add comes later (rb_session_start)
        s->src_ch[r] = (uint8_t)d.channels;
        s->max_src_ch = std::max<uint32_t>(s->max_src_ch, d.channels);
        s->prog_op0[r] = (uint32_t)s->prog_ops.size(), s->prog_n[r] = (uint32_t)progs[i].size(), s->no_silence[r] = no_silence[i];
        s->prog_ops.insert(s->prog_ops.end(), progs[i].begin(), progs[i].end());
        if (take_n[i] != ~0ull) {   // the take's last frame, padded: the source ends there
            s->prog_end[r] = (take_n[i] + d.channels - 1) / d.channels;
            if (s->prog_end[r] == 0) s->st[r].eof = true;
        }
        s->gen_of[r] = gen[i] ? (uint32_t)s->gens.size() : ~0u;
        if (gen[i]) {   // ns[0]: `.take(n)`, the samples the source has; UINT64_MAX: the endless generator
            s->gens.push_back((uint32_t)r), s->gen_fn.push_back(d.effects[0].u32[0]), s->gen_step.push_back(gen_step[i]);
            s->gen_end.push_back(d.effects[0].ns[0]);
            if (d.effects[0].ns[0] == 0) s->st[r].eof = true;
        }
    }
    s->has_prog = !s->prog_ops.empty();
    s->has_biquad = any_biquad;
    // slot rows, in the caller's order, then stably partitioned into classes
    const uint32_t C = s->channels;
    std::vector<rb_session::Slot> slots;
    std::vector<uint32_t> rfrom, rto, rkey;
    for (size_t i = 0; i < n; i++) {
        const uint32_t r = s->pos[i], ci = chs[i];
        auto add = [&](uint32_t ch0, uint32_t w, uint32_t cin) {
            slots.push_back({r, (uint8_t)ch0, (uint8_t)w, (uint8_t)cin});
            rfrom.push_back(from[i]), rto.push_back(to[i]);
            rkey.push_back((key[i] & 0x700u) << 8 | cin | w << 2 | ch0 << 4);   // chain variant, slot
        };
        if (ci == 1 && C >= 2) add(0, 2, 1);
        else
            for (uint32_t c0 = 0, k = std::min(ci, C); c0 < k; c0 += 2) add(c0, std::min(2u, k - c0), std::min(2u, k - c0));
        if (!(ci == 1 && C >= 2) && (ci > 2 || ci > C)) s->plain = false;
    }
    if (slots.size() > 0x7FFFFFFFull) return fail(RB_ERR_INVALID_ARGUMENT, "more than 2^31 slot rows");
    const size_t nr = slots.size();
    s->rows_of.assign(n, {});
    std::vector<uint32_t> gslot;   // per partial row
    uint32_t max_ci = 1;
    for (const auto& cls : lanes::classes_by_ratio(rfrom.data(), rto.data(), rkey.data(), (uint32_t)nr)) {
        rb_session::Class c;
        const rb_session::Slot& s0 = slots[cls[0]];
        const uint32_t src_key = rkey[cls[0]] >> 8;
        c.first = (uint32_t)s->rows.size(), c.count = (uint32_t)cls.size(), c.ch_in = s0.ci, c.ch_out = s0.w;
        c.front = (src_key & 0x400u) != 0;
        c.has_biquad = (src_key & 0x100u) != 0 || c.front, c.has_pre = (src_key & 0x200u) != 0;
        c.ff2 = c.has_biquad;
        for (uint32_t q : cls) {
            c.ff2 = c.ff2 && row_ff2[slots[q].src];
            s->rows_of[slots[q].src].push_back((uint32_t)s->rows.size());
            s->rows.push_back(slots[q]);
        }
        for (uint32_t g = 0; g < (c.count + 31) / 32; g++) gslot.push_back((uint32_t)s0.ch0 | (uint32_t)s0.w << 16);
        max_ci = std::max<uint32_t>(max_ci, s0.ci);
        s->classes.push_back(c);
    }
    RB_CUDA(cudaSetDevice(ctx->device));
    s->n_groups = (uint32_t)gslot.size();
#if defined(RB_SIMT_EMULATE)
    s->emu_fast_tiles.assign(s->classes.size(), 0);
#endif
    s->stride = align_up((size_t)fifo_frames * max_ci + 16, 32);
    // every product below stays far inside 64 bits: rows < 2^31, stride < 2^34 floats, max_block_frames < 2^32
    if ((uint64_t)nr * s->stride > (1ull << 40) || (uint64_t)max_block_frames * C * (s->n_groups + 1) > (1ull << 40))
        return fail(RB_ERR_OUT_OF_MEMORY, "session of this size (sources x fifo_frames, or max_block_frames) exceeds 4 TB of device memory");
    const size_t arena = nr * s->stride * sizeof(float);
    const uint64_t pstride = lanes::round_up_tile((uint64_t)max_block_frames * C);
    RB_CUDA(cudaMalloc(&s->d_fifo[0], arena));
    RB_CUDA(cudaMalloc(&s->d_fifo[1], arena));
    RB_CUDA(cudaMalloc(&s->d_state, nr * 8 * sizeof(float)));
    RB_CUDA(cudaMalloc(&s->d_zeros, 256));
    RB_CUDA(cudaMalloc(&s->d_partial, (size_t)s->n_groups * pstride * sizeof(float)));
    RB_CUDA(cudaMalloc(&s->d_out, pstride * sizeof(float)));
    RB_CUDA(cudaMalloc(&s->d_flags, nr * sizeof(uint32_t)));
    RB_CUDA(cudaMalloc(&s->d_rows, nr * sizeof(lanes::Row)));
    RB_CUDA(cudaMalloc(&s->d_u32, 2 * nr * sizeof(uint32_t)));
    RB_CUDA(cudaMalloc(&s->d_slot, s->n_groups * sizeof(uint32_t)));
    RB_CUDA(cudaMalloc(&s->d_jobs, nr * sizeof(rb_fifo_job)));
    RB_CUDA(cudaMallocHost(&s->h_rows, nr * sizeof(lanes::Row)));
    RB_CUDA(cudaMallocHost(&s->h_u32, 2 * nr * sizeof(uint32_t)));
    RB_CUDA(cudaMallocHost(&s->h_jobs, nr * sizeof(rb_fifo_job)));
    RB_CUDA(cudaMallocHost(&s->h_out, pstride * sizeof(float)));
    RB_CUDA(cudaMemsetAsync(s->d_fifo[0], 0, arena, ctx->stream));
    RB_CUDA(cudaMemsetAsync(s->d_fifo[1], 0, arena, ctx->stream));
    RB_CUDA(cudaMemsetAsync(s->d_state, 0, nr * 8 * sizeof(float), ctx->stream));
    RB_CUDA(cudaMemsetAsync(s->d_zeros, 0, 256, ctx->stream));
    RB_CUDA(cudaMemsetAsync(s->d_flags, 0, nr * sizeof(uint32_t), ctx->stream));
    RB_CUDA(cudaMemcpyAsync(s->d_slot, gslot.data(), s->n_groups * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    if (s->has_prog) {   // the program table goes to the device once; every push of such a session carries program jobs
        RB_CUDA(cudaMalloc(&s->d_prog, s->prog_ops.size() * sizeof(rb_prog_op)));
        RB_CUDA(cudaMalloc(&s->d_pjobs, nr * sizeof(rb_fifo_prog_job)));
        RB_CUDA(cudaMallocHost(&s->h_pjobs, nr * sizeof(rb_fifo_prog_job)));
        RB_CUDA(cudaMemcpyAsync(s->d_prog, s->prog_ops.data(), s->prog_ops.size() * sizeof(rb_prog_op), cudaMemcpyHostToDevice, ctx->stream));
    }
    if (!s->gens.empty()) {   // every generator starts at phase 0.0 (signal_generator.rs:126)
        const size_t ng = s->gens.size();
        for (int k = 0; k < 2; k++) RB_CUDA(cudaMalloc(&s->d_phase[k], ng * sizeof(float)));
        RB_CUDA(cudaMalloc(&s->d_gjobs, ng * sizeof(rb_fifo_gen_job)));
        RB_CUDA(cudaMallocHost(&s->h_gjobs, ng * sizeof(rb_fifo_gen_job)));
        RB_CUDA(cudaMemsetAsync(s->d_phase[0], 0, ng * sizeof(float), ctx->stream));
    }
    RB_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = s.release();
    return RB_OK;
}

// The staging buffer of the pushes: every source's FIFO capacity in its own interleaving.
static cudaError_t session_staging(rb_session* s) {
    if (s->d_stage) return cudaSuccess;
    return cudaMalloc(&s->d_stage, s->st.size() * (size_t)s->fifo_cap * s->max_src_ch * sizeof(float));
}
// Scatter jobs for `frames` new frames of source r (source order) at float offset `src` of the staging buffer, appended to
// h_jobs from index j on; returns the new job count.
static uint32_t session_jobs(rb_session* s, size_t r, uint64_t src, uint64_t frames, uint32_t j) {
    for (uint32_t q : s->rows_of[r]) {
        const rb_session::Slot& sl = s->rows[q];
        const rb_fifo_job job{src, q, (uint32_t)frames, (uint32_t)s->st[r].fill(), s->src_ch[r], sl.ch0, sl.ci, 0};
        if (s->has_prog) s->h_pjobs[j++] = rb_fifo_prog_job{job, s->prog_pos[r], s->prog_op0[r], s->prog_n[r]};
        else s->h_jobs[j++] = job;
    }
    return j;
}
static cudaError_t session_scatter(rb_session* s, uint32_t n_jobs, cudaStream_t stq) {
    cudaError_t e;
    if (s->has_prog) {
        e = cudaMemcpyAsync(s->d_pjobs, s->h_pjobs, n_jobs * sizeof(rb_fifo_prog_job), cudaMemcpyHostToDevice, stq);
        return e != cudaSuccess ? e : rb_lanes_fifo_scatter_prog(s->d_stage, s->d_pjobs, n_jobs, s->d_prog, s->d_fifo[s->cur], s->stride, s->d_flags, stq);
    }
    e = cudaMemcpyAsync(s->d_jobs, s->h_jobs, n_jobs * sizeof(rb_fifo_job), cudaMemcpyHostToDevice, stq);
    return e != cudaSuccess ? e : rb_lanes_fifo_scatter(s->d_stage, s->d_jobs, n_jobs, s->d_fifo[s->cur], s->stride, s->d_flags, stq);
}
// A take has ended source r (source order): rodio stops pulling its input, so whatever is pushed later is dropped.
static bool session_take_ended(const rb_session* s, size_t r) { return s->prog_pos[r] >= s->prog_end[r]; }
// Frames of a push of n frames into source r that its take lets through (all of them without a take).
static uint64_t session_take_room(const rb_session* s, size_t r, uint64_t n) {
    return std::min(n, s->prog_end[r] - std::min(s->prog_end[r], s->prog_pos[r]));
}
// The frames the source's take still lets through (~0: no take).
static uint64_t session_take_left(const rb_session* s, size_t r) {
    return s->prog_end[r] == ~0ull ? ~0ull : s->prog_end[r] - std::min(s->prog_end[r], s->prog_pos[r]);
}
// After `frames` frames went into source r: its program index advances; the take's last frame ends the source.  `changes`: what
// the push's span marks do to its runs (session_span_changes; checked by session_runs_ok beforehand).
static void session_pushed(rb_session* s, size_t r, uint64_t frames, const std::vector<session::CapChange>& changes = {}) {
    session::schedule_push(s->st[r], frames, session_take_left(s, r), true, changes.data(), changes.size());
    s->has_sched = s->has_sched || s->st[r].run_cap != 0;
    s->st[r].pushed += frames;
    s->prog_pos[r] += frames;
    if (session_take_ended(s, r)) s->st[r].eof = true;
}
// Generators that have not ended hold what their FIFO takes, as far as their take and `.take(n)` let them through, as if those
// frames had been pushed: every generator's share of the next fill goes into h_gjobs (frames 0: its phase passes through) and
// through session_pushed; gen_frames counts the samples.  Host bookkeeping only -- session_render_block launches the fill, and
// callers that do not render put the streams back (session_gen_undo).
struct SessionGenUndo {
    std::vector<session::Stream> st;
    std::vector<uint64_t> prog_pos;
    bool has_sched = false;
};
static SessionGenUndo session_gen_top_up(rb_session* s) {
    SessionGenUndo u;
    s->gen_frames = 0;
    if (s->gens.empty()) return u;
    u.st = s->st, u.prog_pos = s->prog_pos, u.has_sched = s->has_sched;
    for (uint32_t g = 0; g < (uint32_t)s->gens.size(); g++) {
        const size_t r = s->gens[g];
        session::Stream& st = s->st[r];
        const uint64_t k = st.eof ? 0 : std::min({(uint64_t)s->fifo_cap - st.fill(), session_take_left(s, r), s->gen_end[g] - s->prog_pos[r]});
        s->h_gjobs[g] = rb_fifo_gen_job{s->prog_pos[r], s->rows_of[r][0], (uint32_t)st.fill(), (uint32_t)k, g, s->prog_op0[r], s->prog_n[r], s->gen_fn[g], s->gen_step[g]};
        if (k) session_pushed(s, r, k);
        if (s->prog_pos[r] >= s->gen_end[g]) st.eof = true;
        s->gen_frames += k;
    }
    return u;
}
static void session_gen_undo(rb_session* s, SessionGenUndo& u) {
    if (s->gens.empty()) return;
    s->st = std::move(u.st), s->prog_pos = std::move(u.prog_pos), s->has_sched = u.has_sched, s->gen_frames = 0;
}
// The run cap (frames) a report of `span_len` samples gives source r (source order): min(span_len, 32768) samples
// (src/source/uniform.rs:55), BAD_CAP when that is not whole frames or under two; for None the take's cap, or none.
static uint64_t session_report_cap(const rb_session* s, size_t r, uint64_t span_len) {
    if (!span_len) return s->none_cap[r];
    const uint64_t ch = s->src_ch[r], len = std::min<uint64_t>(span_len, RB_UNIFORM_SPAN_CAP);
    return len % ch || len / ch < 2 ? session::BAD_CAP : len / ch;
}
// The span marks of one push into source r (source order) of n_frames frames: validated, and turned into the run caps they give
// from the frame of the push at which a bootstrap first sees them (a mark at sample `at` counts for a bootstrap after at samples or
// more).  A source that does not follow marks keeps only the report.  A run under a report must be whole frames and two of them at
// least; that is checked where a run begins (session_runs_ok), so a report no bootstrap sees is never refused.
static rb_status session_span_changes(const rb_session* s, size_t r, uint64_t n_frames, const rb_span_mark* marks, uint32_t n_marks,
                                      std::vector<session::CapChange>* out) {
    out->clear();
    if (!n_marks) return RB_OK;
    if (!s->restarts) return fail(RB_ERR_STATE, "span marks: the session was created without RB_SESSION_RESTARTS");
    if (!marks) return fail(RB_ERR_INVALID_ARGUMENT, "span marks: marks is NULL");
    const uint64_t ch = s->src_ch[r];
    for (uint32_t k = 0; k < n_marks; k++) {
        if (marks[k].pad_ != 0 || marks[k].at >= n_frames * ch || (k && marks[k].at <= marks[k - 1].at))
            return fail(RB_ERR_INVALID_ARGUMENT, "span marks: `at` must increase strictly and stay inside the push, pad_ must be 0");
        if (!s->follows_marks[r]) continue;
        out->push_back(session::CapChange{(marks[k].at + ch - 1) / ch, session_report_cap(s, r, marks[k].span_len)});
    }
    return RB_OK;
}
// Would the runs a push of `frames` frames (real: PCM, else a pause's silence) begins into source r be served?
static bool session_runs_ok(const rb_session* s, size_t r, uint64_t frames, bool real, const std::vector<session::CapChange>& changes = {}) {
    if (!s->marked && changes.empty()) return true;   // without marks every run cap was checked when the session was created
    session::Stream t = s->st[r];
    return session::schedule_push(t, frames, session_take_left(s, r), real, changes.data(), changes.size());
}
static rb_status session_push_one(rb_session* s, size_t stream, const float* pcm, uint64_t n_frames, const rb_span_mark* marks,
                                  uint32_t n_marks, int end_of_stream) {
    if (!s || (!pcm && n_frames)) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    stream = s->pos[stream];   // class order from here on
    if (s->gen_of[stream] != ~0u && (n_frames || n_marks || end_of_stream)) return fail(RB_ERR_STATE, "a generator source takes no pushes");
    session::Stream& st = s->st[stream];
    std::vector<session::CapChange> changes;
    rb_status rc = session_span_changes(s, stream, n_frames, marks, n_marks, &changes);
    if (rc != RB_OK) return rc;
    if (st.eof) return n_frames && !session_take_ended(s, stream) ? fail(RB_ERR_STATE, "push after end_of_stream") : RB_OK;
    const uint64_t take = session_take_room(s, stream, n_frames);
    if (take > s->fifo_cap - st.fill()) return fail(RB_ERR_BUFFER_TOO_SMALL, "the stream's FIFO is full: render first");
    if (!session_runs_ok(s, stream, take, true, changes))
        return fail(RB_ERR_UNSUPPORTED, "span marks: a converter run would begin that is not whole frames of the source, or shorter than two");
    RB_CUDA(cudaSetDevice(s->ctx->device));
    if (take) {
        // one stream: into the staging buffer, scattered over the FIFOs of its rows
        cudaStream_t stq = s->ctx->stream;
        RB_CUDA(session_staging(s));
        RB_CUDA(cudaMemcpyAsync(s->d_stage, pcm, take * s->src_ch[stream] * sizeof(float), cudaMemcpyHostToDevice, stq));
        RB_CUDA(session_scatter(s, session_jobs(s, stream, 0, take, 0), stq));
        RB_CUDA(cudaStreamSynchronize(stq));   // the caller may reuse `pcm` as soon as we return
        session_pushed(s, stream, take, changes);
    }
    if (n_marks) s->report[stream] = marks[n_marks - 1].span_len, s->marked = true;
    if (end_of_stream) st.eof = true;
    return RB_OK;
}

extern "C" rb_status rb_session_push(rb_session* s, size_t stream, const float* pcm, uint64_t n_frames, int end_of_stream) {
    return session_push_one(s, stream, pcm, n_frames, nullptr, 0, end_of_stream);
}

extern "C" rb_status rb_session_push_spans(rb_session* s, size_t stream, const float* pcm, uint64_t n_frames, const rb_span_mark* marks,
                                           uint32_t n_marks, int end_of_stream) {
    return session_push_one(s, stream, pcm, n_frames, marks, n_marks, end_of_stream);
}

extern "C" rb_status rb_session_push_silence(rb_session* s, size_t stream, uint64_t n_frames) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    const size_t r = s->pos[stream];
    session::Stream& st = s->st[r];
    if (s->gen_of[r] != ~0u)   // its FIFO runs ahead of the converter: zeros appended there would land fifo_frames late
        return fail(RB_ERR_UNSUPPORTED, "silence into a generator source");
    if (st.front)   // rodio does not pull that filter while paused; the render would run it over the zeros
        return fail(RB_ERR_UNSUPPORTED, "silence into a source with a filter in front of the conversion");
    if (s->no_silence[r] && !st.eof)   // rodio's conversion counts the zeros against the take's span and restarts early
        return fail(RB_ERR_UNSUPPORTED, "silence into a source whose take is in front of a resampling conversion");
    if (st.eof) return n_frames && !session_take_ended(s, r) ? fail(RB_ERR_STATE, "silence after end_of_stream") : RB_OK;
    if (n_frames > s->fifo_cap - st.fill()) return fail(RB_ERR_BUFFER_TOO_SMALL, "the stream's FIFO is full: render first");
    if (n_frames == 0) return RB_OK;
    if (!session_runs_ok(s, r, n_frames, false))
        return fail(RB_ERR_UNSUPPORTED, "silence: a converter run would begin under a span report that is not whole frames, or under two");
    RB_CUDA(cudaSetDevice(s->ctx->device));
    cudaStream_t stq = s->ctx->stream;
    for (uint32_t q : s->rows_of[r]) {   // literal +0.0 behind the program: inside the exact-reciprocal class, no flag to set
        const uint32_t ci = s->rows[q].ci;
        RB_CUDA(cudaMemsetAsync(s->d_fifo[s->cur] + q * s->stride + st.fill() * ci, 0, n_frames * ci * sizeof(float), stq));
    }
    RB_CUDA(cudaStreamSynchronize(stq));
    session::schedule_push(st, n_frames, session_take_left(s, r), false);
    st.pushed += n_frames;   // the program's index stands still
    return RB_OK;
}

static rb_status session_push_many(rb_session* s, const float* pcm, const uint64_t* n_frames, const uint8_t* end_of_stream, const uint32_t* n_marks,
                                   const rb_span_mark* marks) {
    if (!s || !n_frames) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    const size_t ns = s->st.size();
    uint64_t total = 0;
    std::vector<uint64_t> take(ns);   // per caller's index: the frames the source's take lets through
    std::vector<std::vector<session::CapChange>> changes(n_marks ? ns : 0);
    for (size_t i = 0, m = 0; i < ns; i++) {   // i: the caller's index, pos[i]: class order
        const session::Stream& st = s->st[s->pos[i]];
        if (s->gen_of[s->pos[i]] != ~0u && (n_frames[i] || (end_of_stream && end_of_stream[i]) || (n_marks && n_marks[i])))
            return fail(RB_ERR_STATE, "stream " + std::to_string(i) + ": a generator source takes no pushes");
        if (n_marks) {
            rb_status rc = session_span_changes(s, s->pos[i], n_frames[i], marks ? marks + m : nullptr, n_marks[i], &changes[i]);
            if (rc != RB_OK) return fail(rc, "stream " + std::to_string(i) + ": " + rb_last_error());
            m += n_marks[i];
        }
        if (st.eof && n_frames[i] && !session_take_ended(s, s->pos[i])) return fail(RB_ERR_STATE, "stream " + std::to_string(i) + ": push after end_of_stream");
        take[i] = st.eof ? 0 : session_take_room(s, s->pos[i], n_frames[i]);
        if (take[i] > s->fifo_cap - st.fill()) return fail(RB_ERR_BUFFER_TOO_SMALL, "stream " + std::to_string(i) + ": FIFO full, render first");
        if (!session_runs_ok(s, s->pos[i], take[i], true, n_marks ? changes[i] : std::vector<session::CapChange>{}))
            return fail(RB_ERR_UNSUPPORTED, "stream " + std::to_string(i) + ": span marks: a converter run would begin that is not whole frames of the source, or shorter than two");
        total += n_frames[i];
    }
    if (total && !pcm) return fail(RB_ERR_INVALID_ARGUMENT, "pcm is NULL");
    RB_CUDA(cudaSetDevice(s->ctx->device));
    if (total) {
        RB_CUDA(session_staging(s));
        cudaStream_t stq = s->ctx->stream;
        // Only the frames kept go to the staging buffer, which holds a full FIFO per source: what a take cuts off (or drops
        // after it has ended) is not bounded by the FIFO.  Without such a cut the packed buffer is staged as it is, in one copy.
        bool cut = false;
        for (size_t i = 0; i < ns; i++) cut = cut || take[i] != n_frames[i];
        uint64_t off = 0, staged = 0;   // floats, in the caller's buffer and in the staging buffer: every source counts its own channels
        uint32_t n_jobs = 0;
        for (size_t i = 0; i < ns; i++) {
            const size_t r = s->pos[i];
            if (take[i]) {
                n_jobs = session_jobs(s, r, staged, take[i], n_jobs);
                if (cut) RB_CUDA(cudaMemcpyAsync(s->d_stage + staged, pcm + off, take[i] * s->src_ch[r] * sizeof(float), cudaMemcpyHostToDevice, stq));
            }
            off += n_frames[i] * s->src_ch[r], staged += take[i] * s->src_ch[r];
        }
        if (!cut) RB_CUDA(cudaMemcpyAsync(s->d_stage, pcm, off * sizeof(float), cudaMemcpyHostToDevice, stq));
        RB_CUDA(session_scatter(s, n_jobs, stq));
        RB_CUDA(cudaStreamSynchronize(stq));
    }
    for (size_t i = 0, m = 0; i < ns; i++) {
        if (n_marks) {
            session_pushed(s, s->pos[i], take[i], changes[i]);
            if (n_marks[i]) s->report[s->pos[i]] = marks[m + n_marks[i] - 1].span_len, s->marked = true;
            m += n_marks[i];
        } else {
            session_pushed(s, s->pos[i], take[i]);
        }
        if (end_of_stream && end_of_stream[i]) s->st[s->pos[i]].eof = true;
    }
    return RB_OK;
}

extern "C" rb_status rb_session_push_packed(rb_session* s, const float* pcm, const uint64_t* n_frames, const uint8_t* end_of_stream) {
    return session_push_many(s, pcm, n_frames, end_of_stream, nullptr, nullptr);
}

extern "C" rb_status rb_session_push_packed_spans(rb_session* s, const float* pcm, const uint64_t* n_frames, const uint8_t* end_of_stream,
                                                  const uint32_t* n_marks, const rb_span_mark* marks) {
    if (s && !n_marks) return fail(RB_ERR_INVALID_ARGUMENT, "n_marks is NULL");
    return session_push_many(s, pcm, n_frames, end_of_stream, n_marks, marks);
}

extern "C" rb_status rb_session_start(rb_session* s, size_t stream) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    session::start(s->st[s->pos[stream]], s->T);   // joins at the frame rendered next; no-op when it is playing already
    return RB_OK;
}

extern "C" rb_status rb_session_follow(rb_session* s, size_t stream, size_t predecessor) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (stream >= s->st.size() || predecessor >= s->st.size() || stream == predecessor)
        return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    session::Stream& st = s->st[s->pos[stream]];
    if (!st.held) return fail(RB_ERR_STATE, "only a source declared with RB_SESSION_HELD can be queued");
    st.follows = (int64_t)s->pos[predecessor];
    return RB_OK;
}

extern "C" rb_status rb_session_skip(rb_session* s, size_t stream) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    session::skip(s->st[s->pos[stream]]);
    return RB_OK;
}

extern "C" rb_status rb_session_set_amplify(rb_session* s, size_t stream, float factor) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    if (s->pads[s->pos[stream]] && !std::isfinite(factor))
        return fail(RB_ERR_UNSUPPORTED, "the source's conversion pads channels with 0.0: its gain behind the conversion stays finite");
    s->post[s->pos[stream]] = factor;
    s->has_post = true;   // sources without an AMPLIFY keep the factor 1.0: x * 1.0 is exact
    return RB_OK;
}

extern "C" rb_status rb_session_set_volume(rb_session* s, size_t stream, float factor) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    const size_t r = s->pos[stream];
    if ((s->pads[r] & 2) && !std::isfinite(factor))
        return fail(RB_ERR_UNSUPPORTED, "the source's take ends inside a frame: the gain in front of the conversion stays finite");
    if (s->st[r].front) {
        s->mid[r] = factor;   // the gain behind a filter in front is always applied
        return RB_OK;
    }
    const uint32_t q = s->rows_of[r][0];
    for (const auto& c : s->classes)
        if (q >= c.first && q < c.first + c.count && !c.has_pre)
            return fail(RB_ERR_STATE, "the source was declared without an AMPLIFY in front of the conversion (declare one with factor 1.0)");
    s->pre[r] = factor;
    return RB_OK;
}

extern "C" rb_status rb_session_set_master(rb_session* s, const rb_effect* effects, uint32_t n_effects) {
    if (!s) return fail(RB_ERR_INVALID_ARGUMENT, "session is NULL");
    if (s->T > 0) return fail(RB_ERR_STATE, "the master chain is set before the first rendered frame");
    rb_master_params p{};
    rb_status st = parse_master(effects, n_effects, s->mixer_rate, &p);
    if (st != RB_OK) return st;
    if (n_effects == 0) {
        s->has_master = false;
        return RB_OK;
    }
    RB_CUDA(cudaSetDevice(s->ctx->device));
    const size_t ns = s->st.size();
    if (!s->d_master[0]) {
        for (int k = 0; k < 2; k++) RB_CUDA(cudaMalloc(&s->d_master[k], 2 * RB_MAX_CHANNELS * sizeof(float)));
        RB_CUDA(cudaMalloc(&s->d_master_runs, ns * sizeof(rb_master_run)));
        RB_CUDA(cudaMallocHost(&s->h_master_runs, ns * sizeof(rb_master_run)));
    }
    RB_CUDA(cudaMemsetAsync(s->d_master[s->master_k], 0, 2 * RB_MAX_CHANNELS * sizeof(float), s->ctx->stream));
    RB_CUDA(cudaStreamSynchronize(s->ctx->stream));
    s->master = p, s->has_master = true;
    return RB_OK;
}

extern "C" rb_status rb_session_available(rb_session* s, uint64_t* frames, int* ended) {
    if (!s || !frames) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    bool e = false;
    SessionGenUndo u = session_gen_top_up(s);   // generators count with the frames the next render gives them
    session::resolve_queue(s->st, s->T);
    *frames = session::renderable(s->st, s->T, ~0ull >> 1, &e);
    if (ended) *ended = e ? 1 : 0;
    session_gen_undo(s, u);
    return RB_OK;
}

static rb_status session_render_block(rb_session* s, float* out_host, uint64_t n);

extern "C" rb_status rb_session_render(rb_session* s, float* out_host, uint64_t max_frames, uint64_t* written, int* ended) {
    if (!s || !written) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *written = 0;
    bool e = false;
    SessionGenUndo u = session_gen_top_up(s);   // generators first: a generator never holds the mixer up
    session::resolve_queue(s->st, s->T);   // queued sources whose predecessor's end is known by now get their place on the timeline
    const uint64_t n = session::renderable(s->st, s->T, std::min<uint64_t>(max_frames, s->max_block), &e);
    if (ended) *ended = e ? 1 : 0;
    if (n == 0 || !out_host) {   // nothing is rendered: the generators are topped up by the render that is
        session_gen_undo(s, u);
        return n == 0 ? RB_OK : fail(RB_ERR_INVALID_ARGUMENT, "out_host is NULL");
    }
    if (s->has_sched)
        for (session::Stream& st : s->st) session::settle(st);
    rb_status rc = session_render_block(s, out_host, n);
    if (rc != RB_OK) {
        session_gen_undo(s, u);
        return rc;
    }
    if (s->gen_frames) s->phase_k ^= 1, s->gen_frames = 0;
    *written = n;
    if (ended) {
        bool e2 = false;
        session::renderable(s->st, s->T, 1, &e2);
        *ended = e2 ? 1 : 0;
    }
    return RB_OK;
}

// Room for n_cuts cuts of a block (and the row offsets of the cut lists): grown, never shrunk.
static cudaError_t session_cut_buffers(rb_session* s, size_t n_cuts) {
    cudaError_t e = cudaSuccess;
    if (!s->d_cut_first) {
        const size_t nr = s->rows.size();
        if ((e = cudaMalloc(&s->d_cut_first, (nr + 1) * sizeof(uint32_t))) != cudaSuccess) return e;
        if ((e = cudaMallocHost(&s->h_cut_first, (nr + 1) * sizeof(uint32_t))) != cudaSuccess) return e;
    }
    if (n_cuts <= s->cut_cap) return e;
    const size_t cap = std::max(n_cuts, 2 * s->cut_cap);
    cudaFree(s->d_cuts), cudaFreeHost(s->h_cuts);
    s->d_cuts = nullptr, s->h_cuts = nullptr, s->cut_cap = 0;
    if ((e = cudaMalloc(&s->d_cuts, cap * sizeof(lanes::Cut))) != cudaSuccess) return e;
    if ((e = cudaMallocHost(&s->h_cuts, cap * sizeof(lanes::Cut))) != cudaSuccess) return e;
    s->cut_cap = cap;
    return e;
}

// One launch per class over the frames [T, T + n), which every source can supply; a source may restart any number of times in it.
static rb_status session_render_block(rb_session* s, float* out_host, uint64_t n) {
    RB_CUDA(cudaSetDevice(s->ctx->device));
    cudaStream_t stq = s->ctx->stream;
    const size_t ns = s->st.size(), nr = s->rows.size();
    const uint32_t C = s->channels;
    std::vector<session::Part> parts(ns);
    std::vector<uint8_t> quiet(ns, 0);
    float* fifo = s->d_fifo[s->cur];
    for (size_t r = 0; r < ns; r++) {
        parts[r] = session::part_of(s->st[r], s->T, n);
        if (!s->st[r].front && !(lanes::pre_gain_keeps_class(s->pre[r]) && lanes::pre_gain_keeps_class(s->vol_a[r]) && lanes::pre_gain_keeps_class(s->vol_b[r])))
            quiet[r] = 1;   // its class runs the guarded tile in this block (or, DOWN, slow tiles)
    }
    size_t n_cuts = 0;   // cuts of the block, over all rows
    if (s->has_sched) {
        for (size_t q = 0; q < nr; q++) n_cuts += parts[s->rows[q].src].cuts.size();
        if (n_cuts > 0xFFFFFFFFull) return fail(RB_ERR_OUT_OF_MEMORY, "more than 2^32 converter restarts in one block");
        RB_CUDA(session_cut_buffers(s, n_cuts));
    }
    const bool any_cut = n_cuts != 0;
    for (size_t q = 0, k = 0; q < nr; q++) {   // every row of a source renders the source's part: the rows stay in lock step
        const size_t r = s->rows[q].src;
        const session::Part& p = parts[r];
        lanes::Row& row = s->h_rows[q];
        memset(&row, 0, sizeof(row));
        // positions are relative to the converter run of the block's first output (without a schedule: the whole stream)
        row.in = fifo + q * s->stride, row.L = p.out_len ? p.run_end - s->st[r].i0 : s->st[r].fill(), row.out_len = p.out_len, row.mix_start = p.mix_start;
        row.n_int = p.n_int, row.o0 = p.o0, row.i0 = s->st[r].i0 - p.run_i, row.state = s->d_state + 8 * q;
        if (s->has_sched) {
            s->h_cut_first[q] = (uint32_t)k;
            for (const session::RunCut& c : p.cuts) s->h_cuts[k++] = lanes::Cut{c.m, c.n_int, s->st[r].i0 - c.i, c.end - s->st[r].i0};
            s->h_cut_first[q + 1] = (uint32_t)k;
        }
        const float* co = &s->coef[5 * r];
        row.b0 = co[0], row.b1 = co[1], row.b2 = co[2], row.a1 = co[3], row.a2 = co[4], row.ffk = s->ffk[r];
        row.post = s->post[r], row.pre = s->pre[r], row.mid = s->mid[r];
        row.flags = (p.continues ? lanes::ROW_CONTINUES : 0u) | (quiet[r] ? lanes::ROW_FORCE_SLOW : 0u);
        row.f0 = s->st[r].fpos - s->st[r].i0, row.ga = s->vol_a[r], row.gb = s->vol_b[r];
    }
    RB_CUDA(cudaMemcpyAsync(s->d_rows, s->h_rows, nr * sizeof(lanes::Row), cudaMemcpyHostToDevice, stq));
    if (s->gen_frames) {   // the generators' new frames (session_gen_top_up), in front of the kernels that read them
        const uint32_t ng = (uint32_t)s->gens.size();
        RB_CUDA(cudaMemcpyAsync(s->d_gjobs, s->h_gjobs, ng * sizeof(rb_fifo_gen_job), cudaMemcpyHostToDevice, stq));
        RB_CUDA(rb_lanes_fifo_generate(s->d_gjobs, ng, s->d_prog, s->d_phase[s->phase_k], s->d_phase[s->phase_k ^ 1], fifo, s->stride, s->d_flags, stq));
    }
    if (any_cut) {
        RB_CUDA(cudaMemcpyAsync(s->d_cuts, s->h_cuts, n_cuts * sizeof(lanes::Cut), cudaMemcpyHostToDevice, stq));
        RB_CUDA(cudaMemcpyAsync(s->d_cut_first, s->h_cut_first, (nr + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, stq));
    }
    const uint64_t pstride = lanes::round_up_tile((uint64_t)s->max_block * C);
    // rows of the partial buffer are only written inside each warp's span: clear what this block may read
    RB_CUDA(cudaMemsetAsync(s->d_partial, 0, (size_t)s->n_groups * pstride * sizeof(float), stq));
    uint32_t g0 = 0;
    for (const auto& c : s->classes) {   // one launch per class over its rows and its partial rows
        lanes::Args a{};
        a.rows = s->d_rows + c.first, a.n_rows = c.count, a.n_groups = (c.count + 31) / 32;
        const session::Stream& s0 = s->st[s->rows[c.first].src];
        lanes::fill_ratio(a, s0.from, s0.to, c.ch_out);
        a.mix_len = n, a.pstride = pstride;
        a.partial = s->d_partial + (size_t)g0 * pstride, a.zeros = s->d_zeros, a.unsafe = s->d_flags + c.first;
        bool guard = false, cut = false;   // cut: some row of the class restarts in this block -- the class takes the RESTART twin
        for (uint32_t q = c.first; q < c.first + c.count; q++) {
            guard = guard || quiet[s->rows[q].src];
            cut = cut || (any_cut && s->h_cut_first[q + 1] > s->h_cut_first[q]);
        }
#if defined(RB_SIMT_EMULATE)
        const uint64_t fast0 = simt::g_emu_count[0];
#endif
        if (cut) {
            a.cuts = s->d_cuts, a.cut_first = s->d_cut_first + c.first;
#if defined(RB_SIMT_EMULATE)
            session_host::g_restart_readable.clear();
            for (const auto& b : {std::pair<const void*, size_t>{fifo, nr * s->stride * sizeof(float)}, {s->d_rows, nr * sizeof(lanes::Row)}, {s->d_cuts, n_cuts * sizeof(lanes::Cut)},
                                  {s->d_cut_first, (nr + 1) * sizeof(uint32_t)}, {s->d_state, nr * 8 * sizeof(float)}, {s->d_zeros, 256},
                                  {s->d_flags, nr * sizeof(uint32_t)}})
                session_host::g_restart_readable.push_back({(const char*)b.first, (const char*)b.first + b.second});
#endif
            RB_CUDA(rb_lanes_launch_restart(a, c.ch_in, c.ch_out, c.has_biquad, c.front, stq));
            s->restart_launches++;
        } else {
            RB_CUDA(rb_lanes_launch_kernel(a, c.ch_in, c.ch_out, c.has_biquad, c.ff2, s->has_post, c.has_pre, c.front, guard, stq));
        }
#if defined(RB_SIMT_EMULATE)
        s->emu_fast_tiles[&c - s->classes.data()] += simt::g_emu_count[0] - fast0;
#endif
        g0 += a.n_groups;
    }
    RB_CUDA(rb_lanes_launch_sum_slots(s->d_partial, s->d_slot, s->n_groups, pstride, n, C, s->d_out, stq));
    if (s->has_master) {
        // the block's active runs: frames some source covers.  A frame no source covers (a source declared to join later, the
        // others ended) is a gap: MixerSource::next() is None there, the chain is not pulled and the frame stays 0.0.
        std::vector<std::pair<uint64_t, uint64_t>> iv;
        for (size_t r = 0; r < ns; r++)
            if (parts[r].out_len) iv.push_back({parts[r].mix_start, parts[r].mix_start + parts[r].out_len});
        std::sort(iv.begin(), iv.end());
        uint32_t n_runs = 0;
        uint64_t seq = 0;
        for (size_t i = 0; i < iv.size();) {
            uint64_t lo = iv[i].first, hi = iv[i].second;
            for (i++; i < iv.size() && iv[i].first <= hi; i++) hi = std::max(hi, iv[i].second);
            s->h_master_runs[n_runs++] = {(seq + hi - lo) * C, (lo - seq) * C};
            seq += hi - lo;
        }
        if (n_runs) RB_CUDA(cudaMemcpyAsync(s->d_master_runs, s->h_master_runs, n_runs * sizeof(rb_master_run), cudaMemcpyHostToDevice, stq));
        RB_CUDA(rb_launch_master(s->d_out, s->d_master_runs, n_runs, seq * C, C, s->master, s->d_master[s->master_k], s->d_master[s->master_k ^ 1], stq));
    }
    // the host already knows what every stream consumed: compact the FIFOs into the other arena behind the kernel.
    // The bookkeeping is advanced here and committed by the synchronisation below: when a CUDA call in between fails, the
    // snapshot comes back, so that FIFO positions, volumes and T never run ahead of what the device has done.
    const std::vector<session::Stream> st_before = s->st;
    const std::vector<float> va_before = s->vol_a, vb_before = s->vol_b;
    const uint32_t cur_before = s->cur;
    auto roll_back = [&]() { s->st = st_before, s->vol_a = va_before, s->vol_b = vb_before, s->cur = cur_before; };
#define RB_CUDA_TX(call)                                                                              \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) {                                                                      \
            roll_back();                                                                              \
            return fail(RB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));             \
        }                                                                                             \
    } while (0)
    for (size_t r = 0; r < ns; r++) {
        const uint64_t fill_before = s->st[r].fill(), pulled_before = s->st[r].fpos;
        const uint64_t drop = session::advance(s->st[r], parts[r]);
        // the frames the converter pulled in this block carry the block's factor from now on
        const float vol = s->st[r].front ? s->mid[r] : s->pre[r];
        const uint64_t pulled = s->st[r].fpos - pulled_before;
        if (pulled >= 2) s->vol_a[r] = s->vol_b[r] = vol;
        else if (pulled == 1) s->vol_a[r] = s->vol_b[r], s->vol_b[r] = vol;
        for (uint32_t q : s->rows_of[r]) {   // floats
            const uint32_t ci = s->rows[q].ci;
            s->h_u32[q] = (uint32_t)(drop * ci), s->h_u32[nr + q] = (uint32_t)((fill_before - drop) * ci);
        }
    }
    RB_CUDA_TX(cudaMemcpyAsync(s->d_u32, s->h_u32, 2 * nr * sizeof(uint32_t), cudaMemcpyHostToDevice, stq));
    RB_CUDA_TX(rb_lanes_fifo_compact(fifo, s->d_fifo[s->cur ^ 1], s->stride, s->d_u32, s->d_u32 + nr, (uint32_t)nr, stq));
    s->cur ^= 1;
    RB_CUDA_TX(cudaMemcpyAsync(s->h_out, s->d_out, n * C * sizeof(float), cudaMemcpyDeviceToHost, stq));
    RB_CUDA_TX(cudaStreamSynchronize(stq));
#undef RB_CUDA_TX
    if (s->has_master) s->master_k ^= 1;
    memcpy(out_host, s->h_out, n * C * sizeof(float));
    s->T += n;
    return RB_OK;
}

extern "C" rb_status rb_session_source_runs(rb_session* s, size_t stream, uint64_t* runs_started) {
    if (!s || !runs_started) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (stream >= s->st.size()) return fail(RB_ERR_INVALID_ARGUMENT, "stream index out of range");
    *runs_started = session::runs_started(s->st[s->pos[stream]]);
    return RB_OK;
}

extern "C" rb_status rb_session_restart_launches(rb_session* s, uint64_t* launches) {
    if (!s || !launches) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    *launches = s->restart_launches;
    return RB_OK;
}

#if defined(RB_SIMT_EMULATE)
// CPU build only (not in the C ABI): fast tiles the emulator ran for each class of the session so far, in class order; returns
// the number of classes.  Lets the tests show that no layout passes on slow tiles alone.
extern "C" uint32_t rb_session_emu_fast_tiles(const rb_session* s, uint64_t* out, uint32_t cap) {
    for (size_t k = 0; k < s->emu_fast_tiles.size() && k < cap; k++) out[k] = s->emu_fast_tiles[k];
    return (uint32_t)s->emu_fast_tiles.size();
}
#endif

// ---- block-to-block state as a blob ----
// One record per slot row, in class order; the FIFO contents of every row follow the records.  A session whose every source is one
// row carrying all of its channels (mono and stereo mixers, mono sources anywhere) writes version 5; any other layout writes
// version 6, which adds one layout record per row between the records and the FIFO contents, so that a blob only restores a
// session of the same layout.
namespace {
struct SessionBlobHeader {
    uint32_t magic, version, n_streams, has_biquad, channels, pad_;   // n_streams: rows
    uint64_t T;
};
struct SessionBlobStream {   // in class order (the same descriptors give the same order); the source's fields repeat on each of its rows
    uint64_t mix_start, pushed, out_done, i0;
    uint32_t from, to;
    uint32_t eof, unsafe, fill, filter_ahead;   // fill in frames; filter_ahead = fpos - i0 of a filter in front of the conversion
    float state[8];                      // 4 per channel of the row
    float vol_a, vol_b;                  // factor of the two frames in front of fpos (rb_session_set_volume)
    float vol, post;                     // the current factors: rb_session_set_volume / rb_session_set_amplify
    uint32_t held;                       // still waiting for rb_session_start / its predecessor (RB_SESSION_HELD)
    int32_t follows;                     // class-order index of the first row of the source it is queued behind (rb_session_follow), -1: none
};
struct SessionBlobSlot {     // version 6: the row's source (source order) and slot
    uint32_t src, slot;      // slot = ch0 | w << 8 | ci << 16
};
// Behind the FIFO contents when the session has a master chain (header pad_ = 1); without one the blob ends with them.
struct SessionBlobMaster {
    rb_master_params params;             // a blob only restores a session with the same chain
    uint32_t channels;
    float integ[RB_MAX_CHANNELS], peak[RB_MAX_CHANNELS];
};
// Version 7 (a session with push programs): the layout records of every row as in version 6, then one record per source (source
// order) and the program table, then the FIFO contents.  A blob only restores a session with the same programs.
struct SessionBlobProg {
    uint64_t frames;                     // frames of the source that went through its program
    uint32_t op0, n_ops;
};
// Version 8 (a session some source of which has a restart schedule): version 6 or, with push programs, 7, then one run record per
// source (source order), each followed by its n_ends run ends, then the FIFO contents.  A blob only restores a session with the
// same schedules.
// Version 9 (a session some push of which carried span marks): version 8 with the source's report at the pushed end (samples,
// 0: None) behind each run record, in front of its run ends; the run cap is the one that report gives.  It restores into any
// session of the same shape created with RB_SESSION_RESTARTS.
struct SessionBlobRun {
    uint64_t run_cap, run_i, run_o, sched_end, runs_done, n_ends;
};
// Version 10 (a session with generator sources): the blob the session would otherwise write (version 5 to 9, with 10 in its
// header), then one record per generator (phase slot order) and a tail with the version that record carries.  A blob only restores
// a session with the same generators; sessions without generators never write or take version 10.
struct SessionBlobGen {
    uint32_t src, fn;                    // source order; rb_signal_function
    float step, phase;                   // the phase step; the phase of its next sample
    uint64_t generated, end;             // samples generated so far; ns[0] of its descriptor
};
struct SessionBlobGenTail {              // the blob's last bytes
    uint32_t version, n_gens;
};
constexpr uint32_t SESSION_MAGIC = 0x52425353u;   // "RBSS"
uint32_t blob_version(const rb_session* s) { return s->marked ? 9u : s->has_sched ? 8u : s->has_prog ? 7u : s->plain ? 5u : 6u; }
uint64_t blob_run_bytes(const rb_session* s) {
    uint64_t n = 0;
    if (s->has_sched || s->marked)
        for (const session::Stream& st : s->st) n += sizeof(SessionBlobRun) + (s->marked ? sizeof(uint64_t) : 0) + st.ends.size() * sizeof(uint64_t);
    return n;
}
SessionBlobSlot blob_slot(const rb_session::Slot& sl) { return {sl.src, (uint32_t)sl.ch0 | (uint32_t)sl.w << 8 | (uint32_t)sl.ci << 16}; }
// the fields a source's rows share
bool same_source_fields(const SessionBlobStream& a, const SessionBlobStream& b) {
    return a.mix_start == b.mix_start && a.pushed == b.pushed && a.out_done == b.out_done && a.i0 == b.i0 && a.from == b.from && a.to == b.to &&
           a.eof == b.eof && a.fill == b.fill && a.filter_ahead == b.filter_ahead && !memcmp(&a.vol_a, &b.vol_a, 4 * sizeof(float)) &&
           a.held == b.held && a.follows == b.follows;
}
}  // namespace

extern "C" rb_status rb_session_get_state(rb_session* s, void* buf, uint64_t cap, uint64_t* size) {
    if (!s || !size) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    const size_t nr = s->rows.size(), ns = s->st.size();
    const uint64_t n_slots = blob_version(s) == 5u ? 0 : nr;
    const uint64_t prog_bytes = s->has_prog ? ns * sizeof(SessionBlobProg) + s->prog_ops.size() * sizeof(rb_prog_op) : 0;
    uint64_t need = sizeof(SessionBlobHeader) + nr * sizeof(SessionBlobStream) + n_slots * sizeof(SessionBlobSlot) + prog_bytes + blob_run_bytes(s);
    const uint32_t C = s->channels;
    for (size_t q = 0; q < nr; q++) need += s->st[s->rows[q].src].fill() * s->rows[q].ci * sizeof(float);
    if (s->has_master) need += sizeof(SessionBlobMaster);
    const uint64_t inner = need, ng = s->gens.size();
    if (ng) need += ng * sizeof(SessionBlobGen) + sizeof(SessionBlobGenTail);
    *size = need;
    if (!buf) return RB_OK;
    if (cap < need) return fail(RB_ERR_BUFFER_TOO_SMALL, "state buffer too small");
    RB_CUDA(cudaSetDevice(s->ctx->device));
    std::vector<float> state(8 * nr);
    std::vector<uint32_t> flags(nr);
    RB_CUDA(cudaMemcpyAsync(state.data(), s->d_state, 8 * nr * sizeof(float), cudaMemcpyDeviceToHost, s->ctx->stream));
    RB_CUDA(cudaMemcpyAsync(flags.data(), s->d_flags, nr * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->ctx->stream));
    float mstate[2 * RB_MAX_CHANNELS] = {0};
    if (s->has_master)
        RB_CUDA(cudaMemcpyAsync(mstate, s->d_master[s->master_k], 2 * C * sizeof(float), cudaMemcpyDeviceToHost, s->ctx->stream));
    std::vector<float> phase(ng);
    if (ng) RB_CUDA(cudaMemcpyAsync(phase.data(), s->d_phase[s->phase_k], ng * sizeof(float), cudaMemcpyDeviceToHost, s->ctx->stream));
    uint8_t* p = (uint8_t*)buf;
    SessionBlobHeader h{SESSION_MAGIC, ng ? 10u : blob_version(s), (uint32_t)nr, s->has_biquad ? 1u : 0u, C, s->has_master ? 1u : 0u, s->T};
    memcpy(p, &h, sizeof(h)), p += sizeof(h);
    uint8_t* recs = p;
    p += nr * sizeof(SessionBlobStream);
    for (size_t q = 0; q < n_slots; q++) {
        const SessionBlobSlot sl = blob_slot(s->rows[q]);
        memcpy(p, &sl, sizeof(sl)), p += sizeof(sl);
    }
    if (s->has_prog) {
        for (size_t r = 0; r < ns; r++) {
            const SessionBlobProg b{s->prog_pos[r], s->prog_op0[r], s->prog_n[r]};
            memcpy(p, &b, sizeof(b)), p += sizeof(b);
        }
        memcpy(p, s->prog_ops.data(), s->prog_ops.size() * sizeof(rb_prog_op)), p += s->prog_ops.size() * sizeof(rb_prog_op);
    }
    if (s->has_sched || s->marked)
        for (size_t r = 0; r < ns; r++) {
            const session::Stream& st = s->st[r];
            const SessionBlobRun b{st.run_cap, st.run_i, st.run_o, st.sched_end, st.runs_done, st.ends.size()};
            memcpy(p, &b, sizeof(b)), p += sizeof(b);
            if (s->marked) memcpy(p, &s->report[r], sizeof(uint64_t)), p += sizeof(uint64_t);
            memcpy(p, st.ends.data(), st.ends.size() * sizeof(uint64_t)), p += st.ends.size() * sizeof(uint64_t);
        }
    for (size_t q = 0; q < nr; q++) {
        const uint64_t fill = s->st[s->rows[q].src].fill() * s->rows[q].ci;   // floats
        if (fill) RB_CUDA(cudaMemcpyAsync(p, s->d_fifo[s->cur] + q * s->stride, fill * sizeof(float), cudaMemcpyDeviceToHost, s->ctx->stream));
        p += fill * sizeof(float);
    }
    RB_CUDA(cudaStreamSynchronize(s->ctx->stream));
    for (size_t q = 0; q < nr; q++) {
        const size_t r = s->rows[q].src;
        const session::Stream& st = s->st[r];
        const int32_t follows = st.follows < 0 ? -1 : (int32_t)s->rows_of[(size_t)st.follows][0];
        SessionBlobStream b{st.mix_start, st.pushed, st.out_done, st.i0, st.from, st.to, st.eof ? 1u : 0u, flags[q], (uint32_t)st.fill(), (uint32_t)(st.fpos - st.i0), {0}, s->vol_a[r], s->vol_b[r],
                            st.front ? s->mid[r] : s->pre[r], s->post[r], st.held ? 1u : 0u, follows};
        for (uint32_t k = 0; k < 8; k++) b.state[k] = state[8 * q + k];
        memcpy(recs + q * sizeof(b), &b, sizeof(b));
    }
    if (s->has_master) {
        SessionBlobMaster m{};
        m.params = s->master, m.channels = C;
        for (uint32_t c = 0; c < C; c++) m.integ[c] = mstate[c], m.peak[c] = mstate[C + c];
        memcpy(p, &m, sizeof(m));
    }
    if (ng) {
        p = (uint8_t*)buf + inner;
        for (uint32_t g = 0; g < ng; g++) {
            const uint32_t r = s->gens[g];
            const SessionBlobGen b{r, s->gen_fn[g], s->gen_step[g], phase[g], s->prog_pos[r], s->gen_end[g]};
            memcpy(p, &b, sizeof(b)), p += sizeof(b);
        }
        const SessionBlobGenTail tail{blob_version(s), (uint32_t)ng};
        memcpy(p, &tail, sizeof(tail));
    }
    return RB_OK;
}

extern "C" rb_status rb_session_set_state(rb_session* s, const void* buf, uint64_t size) {
    if (!s || !buf) return fail(RB_ERR_INVALID_ARGUMENT, "NULL argument");
    const size_t nr = s->rows.size(), ns = s->st.size();
    const uint64_t prog_bytes = s->has_prog ? ns * sizeof(SessionBlobProg) + s->prog_ops.size() * sizeof(rb_prog_op) : 0;
    const uint8_t* p = (const uint8_t*)buf;
    SessionBlobHeader h;
    if (size < sizeof(h)) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
    memcpy(&h, p, sizeof(h)), p += sizeof(h);
    const uint32_t C = s->channels;
    // version 10: the generator records and the tail come off the end, the rest is read as the version the tail names
    const size_t ng = s->gens.size();
    const bool v10 = h.magic == SESSION_MAGIC && h.version == 10u;
    if (v10 != (ng != 0) && h.magic == SESSION_MAGIC && h.version >= 5u && h.version <= 10u)
        return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with other generator sources");
    std::vector<SessionBlobGen> gens(ng);
    if (v10) {
        const uint64_t tail_bytes = ng * sizeof(SessionBlobGen) + sizeof(SessionBlobGenTail);
        if (size < sizeof(h) + tail_bytes) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
        SessionBlobGenTail tail;
        memcpy(&tail, (const uint8_t*)buf + size - sizeof(tail), sizeof(tail));
        if (tail.n_gens != ng) return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with other generator sources");
        size -= tail_bytes;
        memcpy(gens.data(), (const uint8_t*)buf + size, ng * sizeof(SessionBlobGen));
        for (size_t g = 0; g < ng; g++) {
            const SessionBlobGen& b = gens[g];
            if (b.src != s->gens[g] || b.fn != s->gen_fn[g] || memcmp(&b.step, &s->gen_step[g], sizeof(float)) || b.end != s->gen_end[g] ||
                b.generated > b.end || !(b.phase >= 0.0f && b.phase < 1.0f))
                return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with other generator sources");
        }
        h.version = tail.version;
        if (h.version == 10u) return fail(RB_ERR_INVALID_ARGUMENT, "not a session state blob");
    }
    if (h.magic != SESSION_MAGIC || h.version < 5u || h.version > 9u) return fail(RB_ERR_INVALID_ARGUMENT, "not a session state blob");
    // a version-9 blob (span marks) restores into a session of the same shape with RB_SESSION_RESTARTS, marked or not
    const bool v9 = h.version == 9u;
    if ((v9 ? !s->restarts : h.version != blob_version(s)) || h.n_streams != nr || h.has_biquad != (s->has_biquad ? 1u : 0u) || h.channels != C)
        return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session of another shape");
    const uint64_t n_slots = h.version == 5u ? 0 : nr;
    uint64_t need = sizeof(h) + nr * sizeof(SessionBlobStream) + n_slots * sizeof(SessionBlobSlot) + prog_bytes;
    if (size < need) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
    std::vector<SessionBlobStream> recs(nr);
    memcpy(recs.data(), p, nr * sizeof(SessionBlobStream)), p += nr * sizeof(SessionBlobStream);
    for (size_t q = 0; q < n_slots; q++) {
        SessionBlobSlot sl, mine = blob_slot(s->rows[q]);
        memcpy(&sl, p, sizeof(sl)), p += sizeof(sl);
        if (memcmp(&sl, &mine, sizeof(sl)) != 0) return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session of another layout");
    }
    std::vector<uint64_t> prog_pos(ns, 0);
    if (s->has_prog) {
        for (size_t r = 0; r < ns; r++) {
            SessionBlobProg b;
            memcpy(&b, p, sizeof(b)), p += sizeof(b);
            if (b.op0 != s->prog_op0[r] || b.n_ops != s->prog_n[r] || b.frames > s->prog_end[r])
                return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with other push programs");
            prog_pos[r] = b.frames;
        }
        if (memcmp(p, s->prog_ops.data(), s->prog_ops.size() * sizeof(rb_prog_op)) != 0)
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with other push programs");
        p += s->prog_ops.size() * sizeof(rb_prog_op);
    }
    std::vector<session::Stream> runs(ns);   // the run records, checked against the source's record below
    std::vector<uint64_t> report = s->report;
    if (h.version >= 8u) {
        const uint8_t* const end = (const uint8_t*)buf + size;
        for (size_t r = 0; r < ns; r++) {
            SessionBlobRun b;
            if ((uint64_t)(end - p) < sizeof(b)) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
            memcpy(&b, p, sizeof(b)), p += sizeof(b);
            if (v9) {   // the run cap is the one the report gives, for a source that follows marks and has a schedule
                if ((uint64_t)(end - p) < sizeof(uint64_t)) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
                memcpy(&report[r], p, sizeof(uint64_t)), p += sizeof(uint64_t), need += sizeof(uint64_t);
                const bool eof = recs[s->rows_of[r][0]].eof != 0;   // (a take that has ended takes no more runs, nor their caps)
                if (b.run_cap && s->follows_marks[r] && !eof && b.run_cap != session_report_cap(s, r, report[r]))
                    return fail(RB_ERR_INVALID_ARGUMENT, "state blob: run cap and span report disagree");
            }
            if ((v9 ? !s->follows_marks[r] && b.run_cap : b.run_cap != s->st[r].run_cap) || (!b.run_cap && (b.n_ends || b.run_i || b.run_o)))
                return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with other restart schedules");
            if (b.n_ends > (uint64_t)(end - p) / sizeof(uint64_t)) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
            session::Stream& st = runs[r];
            st.run_cap = b.run_cap, st.run_i = b.run_i, st.run_o = b.run_o, st.sched_end = b.sched_end, st.runs_done = b.runs_done;
            st.ends.resize(b.n_ends);
            memcpy(st.ends.data(), p, b.n_ends * sizeof(uint64_t)), p += b.n_ends * sizeof(uint64_t);
            need += sizeof(b) + b.n_ends * sizeof(uint64_t);
            uint64_t at = b.run_i;   // runs follow one another, none shorter than a frame, the last one the pushes are filling
            for (uint64_t e : st.ends) {
                if (e <= at) return fail(RB_ERR_INVALID_ARGUMENT, "state blob: run record out of order");
                at = e;
            }
            if (!st.ends.empty() && st.ends.back() != b.sched_end) return fail(RB_ERR_INVALID_ARGUMENT, "state blob: run record out of order");
        }
    }
    std::vector<uint8_t> first_row(nr, 0);
    for (const auto& rows : s->rows_of) first_row[rows[0]] = 1;
    for (size_t q = 0; q < nr; q++) {
        const SessionBlobStream& b = recs[q];
        const size_t r = s->rows[q].src;
        if (b.from != s->st[r].from || b.to != s->st[r].to) return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session of another shape");
        if (b.fill > s->fifo_cap || b.pushed - b.i0 != b.fill || (b.i0 & 3u) || b.filter_ahead > b.fill)
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob: FIFO record out of range");
        if (b.follows < -1 || (b.follows >= 0 && ((size_t)b.follows >= nr || !first_row[(size_t)b.follows] || s->rows[(size_t)b.follows].src == r)))
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob: queue record out of range");
        session::Stream chk = runs[r];   // with a schedule: the outputs its runs hold
        chk.from = b.from, chk.to = b.to, chk.pushed = b.pushed, chk.eof = true;
        if (b.out_done > session::out_end(chk) || b.out_done < chk.run_o || chk.run_i > b.pushed)
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob: more outputs rendered than the pushed input holds");
        if (!same_source_fields(b, recs[s->rows_of[r][0]]))
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob: the rows of one source disagree");
        need += (uint64_t)b.fill * s->rows[q].ci * sizeof(float);
    }
    if (h.pad_ != (s->has_master ? 1u : 0u)) return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with another master chain");
    SessionBlobMaster m{};
    if (s->has_master) {
        if (size < need + sizeof(m)) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
        memcpy(&m, (const uint8_t*)buf + need, sizeof(m));
        need += sizeof(m);
        if (m.channels != C || memcmp(&m.params, &s->master, sizeof(m.params)) != 0)
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob belongs to a session with another master chain");
    }
    if (size < need) return fail(RB_ERR_INVALID_ARGUMENT, "state blob truncated");
    if (v10 && size != need) return fail(RB_ERR_INVALID_ARGUMENT, "state blob: generator records out of place");
    for (size_t g = 0; g < ng; g++)   // a generator has received what it generated, less what a skip dropped
        if (recs[s->rows_of[s->gens[g]][0]].pushed > gens[g].generated)
            return fail(RB_ERR_INVALID_ARGUMENT, "state blob: a generator holds more frames than it generated");
    RB_CUDA(cudaSetDevice(s->ctx->device));
    std::vector<float> state(8 * nr);
    std::vector<uint32_t> flags(nr);
    for (size_t r = 0; r < s->st.size(); r++) {   // the source's fields, from its first row
        const SessionBlobStream& b = recs[s->rows_of[r][0]];
        session::Stream& st = s->st[r];
        st.mix_start = b.mix_start, st.pushed = b.pushed, st.out_done = b.out_done, st.i0 = b.i0, st.eof = b.eof != 0, st.fpos = b.i0 + b.filter_ahead, s->vol_a[r] = b.vol_a, s->vol_b[r] = b.vol_b;
        st.held = b.held != 0, st.follows = b.follows < 0 ? -1 : (int64_t)s->rows[(size_t)b.follows].src;
        st.run_i = runs[r].run_i, st.run_o = runs[r].run_o, st.sched_end = runs[r].sched_end, st.runs_done = runs[r].runs_done, st.ends = runs[r].ends;
        if (v9) {   // the report is the state: the cap of the runs the next bootstraps begin follows from it
            st.run_cap = runs[r].run_cap && s->follows_marks[r] && !st.eof ? session_report_cap(s, r, report[r]) : runs[r].run_cap;
            s->has_sched = s->has_sched || st.run_cap != 0;
        }
        (st.front ? s->mid[r] : s->pre[r]) = b.vol;
        if (b.post != s->post[r]) s->post[r] = b.post, s->has_post = true;
    }
    for (size_t q = 0; q < nr; q++) {
        const SessionBlobStream& b = recs[q];
        flags[q] = b.unsafe;
        for (uint32_t k = 0; k < 8; k++) state[8 * q + k] = b.state[k];
        const size_t fill_floats = (size_t)b.fill * s->rows[q].ci;
        if (b.fill) RB_CUDA(cudaMemcpyAsync(s->d_fifo[s->cur] + q * s->stride, p, fill_floats * sizeof(float), cudaMemcpyHostToDevice, s->ctx->stream));
        p += fill_floats * sizeof(float);
    }
    RB_CUDA(cudaMemcpyAsync(s->d_state, state.data(), 8 * nr * sizeof(float), cudaMemcpyHostToDevice, s->ctx->stream));
    RB_CUDA(cudaMemcpyAsync(s->d_flags, flags.data(), nr * sizeof(uint32_t), cudaMemcpyHostToDevice, s->ctx->stream));
    float mstate[2 * RB_MAX_CHANNELS];
    if (s->has_master) {
        for (uint32_t c = 0; c < C; c++) mstate[c] = m.integ[c], mstate[C + c] = m.peak[c];
        RB_CUDA(cudaMemcpyAsync(s->d_master[s->master_k], mstate, 2 * C * sizeof(float), cudaMemcpyHostToDevice, s->ctx->stream));
    }
    std::vector<float> phase(ng);
    for (size_t g = 0; g < ng; g++) phase[g] = gens[g].phase;
    if (ng) RB_CUDA(cudaMemcpyAsync(s->d_phase[s->phase_k], phase.data(), ng * sizeof(float), cudaMemcpyHostToDevice, s->ctx->stream));
    RB_CUDA(cudaStreamSynchronize(s->ctx->stream));
    s->T = h.T;
    if (s->has_prog) s->prog_pos = prog_pos;
    for (size_t g = 0; g < ng; g++) s->prog_pos[s->gens[g]] = gens[g].generated;
    if (v9) s->report = report, s->marked = true;
    return RB_OK;
}
