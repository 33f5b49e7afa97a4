// rodio_b200.hpp — header-only C++ mirror of rodio's `Source` / `Mixer` surface on top of the C ABI
// (include/rodio_b200.h).  rodio is compiled code, so this is the host-side binding a C++ caller links
// against; the Rust shim in bindings/rust/ has the same shape.  Names and argument meaning follow the
// reference (file:line in the comments); where rodio panics this throws std::invalid_argument /
// rodio::Error.  Nothing here touches samples on the CPU: a Source records a PCM buffer and an adapter
// chain, MixerSource drains it through the library in one block.
#pragma once
#include <chrono>
#include <cstdint>
#include <cstring>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "rodio_b200.h"

namespace rodio {

using Sample = float;                       // src/common.rs:36,:48
using Duration = std::chrono::nanoseconds;  // std::time::Duration

struct Error : std::runtime_error {
    rb_status status;
    Error(rb_status s, const std::string& where)
        : std::runtime_error(where + ": " + rb_status_string(s) + " (" + rb_last_error() + ")"), status(s) {}
};
inline void check(rb_status s, const char* where) {
    if (s != RB_OK) throw Error(s, where);
}

// One rb_context per device, shared by everything in the process.
class Context {
  public:
    static rb_context* get(int device = 0) {
        static Context ctx(device);
        return ctx.h_;
    }

  private:
    explicit Context(int device) { check(rb_context_create(device, &h_), "rb_context_create"); }
    ~Context() { rb_context_destroy(h_); }
    rb_context* h_ = nullptr;
};

// AutomaticGainControlSettings — src/source/agc.rs:57-82
struct AutomaticGainControlSettings {
    float target_level = 1.0f;
    Duration attack_time = std::chrono::seconds(4);
    Duration release_time = std::chrono::seconds(0);
    float absolute_max_gain = 7.0f;
};
// LimitSettings — src/source/limit.rs:209-248
struct LimitSettings {
    float threshold = -1.0f;
    float knee_width = 4.0f;
    Duration attack = std::chrono::milliseconds(5);
    Duration release = std::chrono::milliseconds(100);
    LimitSettings with_threshold(float v) const { auto s = *this; s.threshold = v; return s; }
    LimitSettings with_knee_width(float v) const { auto s = *this; s.knee_width = v; return s; }
    LimitSettings with_attack(Duration v) const { auto s = *this; s.attack = v; return s; }
    LimitSettings with_release(Duration v) const { auto s = *this; s.release = v; return s; }
};

// trait Source (src/source/mod.rs:179-759) as a value: PCM + recorded adapters.
class Source {
  public:
    Source(uint16_t channels, uint32_t sample_rate, std::vector<Sample> data, uint32_t span_len)
        : pcm_(std::make_shared<std::vector<Sample>>(std::move(data))), base_channels_(channels), base_rate_(sample_rate),
          span_len_(span_len), channels_(channels), rate_(sample_rate) {
        if (channels == 0 || sample_rate == 0) throw std::invalid_argument("channels / sample_rate are NonZero in rodio");
    }
    uint16_t channels() const { return channels_; }        // Source::channels
    uint32_t sample_rate() const { return rate_; }          // Source::sample_rate

    Source amplify(float value) const { return with(fx(RB_FX_AMPLIFY, {}, {value}, {})); }                 // mod.rs:307-314
    Source amplify_decibel(float value) const { return amplify(rb_db_to_linear(value)); }                  // mod.rs:316-323
    Source speed(float ratio) const {                                                                        // speed.rs:103-133
        Source s = with(fx(RB_FX_SPEED, {}, {ratio}, {}));
        s.rate_ = rb_speed_sample_rate(rate_, ratio);
        return s;
    }
    Source low_pass(uint32_t freq) const { return low_pass_with_q(freq, 0.5f); }                            // mod.rs:686-692
    Source low_pass_with_q(uint32_t freq, float q) const { return with(fx(RB_FX_LOW_PASS, {freq}, {q}, {})); }
    Source high_pass(uint32_t freq) const { return high_pass_with_q(freq, 0.5f); }
    Source high_pass_with_q(uint32_t freq, float q) const { return with(fx(RB_FX_HIGH_PASS, {freq}, {q}, {})); }
    Source reverb(Duration d, float amplitude) const { return with(fx(RB_FX_REVERB, {}, {amplitude}, {ns(d)})); }   // mod.rs:628-634
    Source delay(Duration d) const { return with(fx(RB_FX_DELAY, {}, {}, {ns(d)})); }                        // delay.rs:19-29
    Source distortion(float gain, float threshold) const { return with(fx(RB_FX_DISTORTION, {}, {gain, threshold}, {})); }   // mod.rs:726-731
    Source linear_gain_ramp(Duration d, float start, float end, bool clamp_end) const {                      // mod.rs:534-546
        if (d.count() == 0) throw std::invalid_argument("duration must be greater than zero");
        return with(fx(RB_FX_LINEAR_RAMP, {clamp_end ? 1u : 0u}, {start, end}, {ns(d)}));
    }
    Source fade_in(Duration d) const { return linear_gain_ramp(d, 0.0f, 1.0f, false); }                      // fadein.rs:8-15
    Source fade_out(Duration d) const { return linear_gain_ramp(d, 1.0f, 0.0f, true); }                      // fadeout.rs:8-15
    Source take_duration(Duration d, bool filter_fadeout = false) const {                                    // take.rs:9-26,:89-96
        return with(fx(RB_FX_TAKE_DURATION, {filter_fadeout ? 1u : 0u}, {}, {ns(d)}));
    }
    Source automatic_gain_control(const AutomaticGainControlSettings& s = {}) const {                        // mod.rs:415-446
        return with(fx(RB_FX_AGC, {}, {s.target_level, s.absolute_max_gain, 0.0f}, {ns(s.attack_time), ns(s.release_time)}));
    }
    Source limit(const LimitSettings& s = {}) const {                                                        // limit.rs:94-130
        return with(fx(RB_FX_LIMIT, {}, {s.threshold, s.knee_width}, {ns(s.attack), ns(s.release)}));
    }
    // source::Spatial::new(input, emitter, left_ear, right_ear) — spatial.rs:31-45
    Source spatial(const float (&e)[3], const float (&l)[3], const float (&r)[3]) const {
        Source s = with(fx(RB_FX_SPATIAL, {}, {e[0], e[1], e[2], l[0], l[1], l[2], r[0], r[1], r[2]}, {}));
        s.channels_ = 2;
        return s;
    }
    // source::UniformSourceIterator::new(input, channels, rate) — uniform.rs:33-47
    Source uniform(uint16_t channels, uint32_t rate) const {
        if (channels == 0 || rate == 0) throw std::invalid_argument("target channels / rate must be non-zero");
        Source s = with(fx(RB_FX_UNIFORM, {channels, rate}, {}, {}));
        s.channels_ = channels, s.rate_ = rate;
        return s;
    }

    // Pausable with Player::pause / play at known positions -- pausable.rs:85-97 (RB_FX_PAUSE)
    Source pause_at(uint64_t at_sample, uint64_t n_frames) const { return with(fx(RB_FX_PAUSE, {}, {}, {at_sample, n_frames})); }
    // Source::mix(other) -- mod.rs:253-261, mix.rs:10-53: the second input becomes a descriptor of its own (RB_FX_MIX)
    Source mix(const Source& other) const {
        Source s = with(fx(RB_FX_MIX, {}, {}, {}));
        s.others_.push_back(std::make_shared<Source>(other));
        return s;
    }
    // Source::take_crossfade_with(other, duration) -- mod.rs:444-454 = crossfade.rs:10-23
    Source take_crossfade_with(const Source& other, Duration d) const {
        return take_duration(d, true).mix(other.take_duration(d).fade_in(d));
    }
    // source::from_iter(buffers) -- from_iter.rs:16-27: one source whose format changes from buffer to buffer (RB_FX_APPEND)
    static Source from_iter(const std::vector<Source>& buffers) {
        if (buffers.empty()) throw std::invalid_argument("from_iter of nothing");
        Source s = buffers[0];
        if (!s.effects_.empty()) throw std::invalid_argument("from_iter takes plain buffers");
        for (size_t i = 1; i < buffers.size(); i++) {
            if (!buffers[i].effects_.empty()) throw std::invalid_argument("from_iter takes plain buffers");
            s.effects_.push_back(fx(RB_FX_APPEND, {}, {}, {}));
            s.others_.push_back(std::make_shared<Source>(buffers[i]));
        }
        return s;
    }
    // SignalGenerator::new(sample_rate, frequency, function).take(n) -- signal_generator.rs:85-135: generated on the device.
    // n = UINT64_MAX (the default): the endless generator, which a LiveMixer plays until a take_duration or skip ends it.
    static Source signal_generator(uint32_t sample_rate, float frequency, rb_signal_function f, uint64_t n = UINT64_MAX) {
        if (!(frequency > 0.0f)) throw std::invalid_argument("frequency must be greater than zero");   // :112
        Source s(1, sample_rate, {}, 0);
        s.effects_.push_back(fx(RB_FX_SIGNAL, {(uint32_t)f}, {frequency}, {n}));
        return s;
    }

    // `.collect::<Vec<f32>>()` of this source (its own chain, no mixer conversion)
    std::vector<Sample> collect() const;
    const std::vector<std::shared_ptr<Source>>& others() const { return others_; }
    const std::vector<rb_effect>& effects() const { return effects_; }

    rb_stream_desc desc(uint64_t mix_start = 0) const {
        rb_stream_desc d{};
        d.sample_rate = base_rate_, d.channels = base_channels_, d.format = RB_FMT_F32;
        d.n_samples = pcm_->size(), d.span_len = span_len_;
        d.n_effects = (uint32_t)effects_.size(), d.effects = effects_.data(), d.mix_start = mix_start;
        return d;
    }
    const std::vector<Sample>& pcm() const { return *pcm_; }

  private:
    static uint64_t ns(Duration d) { return (uint64_t)d.count(); }
    static rb_effect fx(uint32_t kind, std::initializer_list<uint32_t> u, std::initializer_list<float> f,
                        std::initializer_list<uint64_t> n) {
        rb_effect e{};
        e.kind = kind;
        size_t i = 0;
        for (uint32_t v : u) e.u32[i++] = v;
        i = 0;
        for (float v : f) e.f32[i++] = v;
        i = 0;
        for (uint64_t v : n) e.ns[i++] = v;
        return e;
    }
    Source with(const rb_effect& e) const {
        Source s = *this;
        s.effects_.push_back(e);
        return s;
    }
    std::shared_ptr<std::vector<Sample>> pcm_;
    uint16_t base_channels_;
    uint32_t base_rate_, span_len_;
    std::vector<rb_effect> effects_;
    std::vector<std::shared_ptr<Source>> others_;   // second inputs of mix() / buffers of from_iter(), one per RB_FX_MIX / RB_FX_APPEND in order
    uint16_t channels_;
    uint32_t rate_;
};

// buffer::SamplesBuffer::new(channels, sample_rate, data) — src/buffer.rs:40-60 (reports its length as the span)
inline Source SamplesBuffer(uint16_t channels, uint32_t sample_rate, std::vector<Sample> data) {
    uint32_t span = (uint32_t)std::min<size_t>(data.size(), 0xFFFFFFFFu);
    return Source(channels, sample_rate, std::move(data), span);
}
// benches/shared.rs TestSource: span-less
inline Source TestSource(std::vector<Sample> data, uint16_t channels, uint32_t sample_rate) {
    return Source(channels, sample_rate, std::move(data), 0);
}

namespace detail {
struct Batch {
    rb_batch* h = nullptr;
    Batch(const std::vector<rb_stream_desc>& descs, uint16_t ch, uint32_t rate, uint32_t flags) {
        check(rb_batch_create(Context::get(), ch, rate, descs.data(), descs.size(), flags, &h), "rb_batch_create");
    }
    ~Batch() { rb_batch_destroy(h); }
};
// The descriptor array of `sources`: the sources themselves, then (breadth first) the second inputs of their mix() adapters and the
// buffers of their from_iter() sequences as descriptors of their own (mix_start = RB_MIX_START_CONSUMED), the adapter that names
// one carrying its index.  Owns the patched effect arrays the descriptors point into.
struct Flat {
    std::vector<const Source*> src;
    std::vector<std::vector<rb_effect>> fx;
    std::vector<rb_stream_desc> descs;
    Flat(const std::vector<const Source*>& sources, const std::vector<uint64_t>& starts) {
        src = sources;
        for (size_t i = 0; i < src.size(); i++) {
            std::vector<rb_effect> e = src[i]->effects();
            size_t k = 0;
            for (rb_effect& x : e)
                if (x.kind == RB_FX_MIX || x.kind == RB_FX_APPEND) {
                    x.u32[0] = (uint32_t)src.size();
                    src.push_back(src[i]->others().at(k++).get());
                }
            fx.push_back(std::move(e));
        }
        for (size_t i = 0; i < src.size(); i++) {
            rb_stream_desc d = src[i]->desc(i < starts.size() ? starts[i] : RB_MIX_START_CONSUMED);
            d.effects = fx[i].data();
            descs.push_back(d);
        }
    }
    void upload(rb_batch* b) const {
        for (size_t i = 0; i < src.size(); i++)
            check(rb_batch_upload(b, i, src[i]->pcm().data(), src[i]->pcm().size()), "rb_batch_upload");
    }
};
}  // namespace detail

inline std::vector<Sample> Source::collect() const {
    detail::Flat flat({this}, {0});
    detail::Batch b(flat.descs, channels_, rate_, RB_KEEP_STREAM_OUTPUTS | RB_NO_FUSION);
    flat.upload(b.h);
    check(rb_batch_render_mix_device(b.h), "rb_batch_render_mix_device");
    uint64_t n = 0, w = 0;
    check(rb_batch_stream_out_len(b.h, 0, &n), "rb_batch_stream_out_len");
    std::vector<Sample> out(n);
    check(rb_batch_read_stream(b.h, 0, out.data(), n, &w), "rb_batch_read_stream");
    out.resize(w);
    return out;
}

namespace mixer {

struct Shared {
    uint16_t channels;
    uint32_t rate;
    std::vector<Source> sources;
    std::vector<uint64_t> starts;
    uint64_t pos = 0;                  // samples MixerSource already handed out
    bool dirty = true;
    std::vector<Sample> rendered;
    std::vector<uint8_t> active;       // position has at least one source playing
    std::vector<rb_effect> rendered_master;   // the MixerSource adapters `rendered` went through
};

// mixer::Mixer — src/mixer.rs:47-66 ; add is infallible like the reference
class Mixer {
  public:
    explicit Mixer(std::shared_ptr<Shared> s) : s_(std::move(s)) {}
    void add(const Source& source) {
        s_->sources.push_back(source);
        s_->starts.push_back(s_->pos);   // joins at the next frame boundary (mixer.rs:175-183), done by the library
        s_->dirty = true;
    }

  private:
    std::shared_ptr<Shared> s_;
};

// mixer::MixerSource — src/mixer.rs:70-136
class MixerSource {
  public:
    explicit MixerSource(std::shared_ptr<Shared> s) : s_(std::move(s)) {}
    uint16_t channels() const { return s_->channels; }
    uint32_t sample_rate() const { return s_->rate; }
    std::optional<size_t> current_span_len() const { return std::nullopt; }
    // Iterator::next — None while no source is playing at this position (mixer.rs:131-135)
    std::optional<Sample> next() {
        render();
        uint64_t p = s_->pos++;
        if (p < s_->rendered.size() && s_->active[p]) return s_->rendered[p];
        return std::nullopt;
    }
    void try_seek(Duration) { throw Error(RB_ERR_NOT_SUPPORTED_SEEK, "MixerSource::try_seek"); }   // mixer.rs:109-113
    // Adapters on the MixerSource itself (rb_batch_set_master): [amplify] [limit] [amplify], over the whole mix.  A new handle
    // on the same mixer, like rodio's adapters that take the source by value.
    MixerSource amplify(float value) const {                                                                // amplify.rs:63-65
        rb_effect e{};
        e.kind = RB_FX_AMPLIFY, e.f32[0] = value;
        return with(e);
    }
    MixerSource limit(const LimitSettings& ls = {}) const {                                                 // limit.rs:94-130
        rb_effect e{};
        e.kind = RB_FX_LIMIT, e.f32[0] = ls.threshold, e.f32[1] = ls.knee_width;
        e.ns[0] = (uint64_t)ls.attack.count(), e.ns[1] = (uint64_t)ls.release.count();
        return with(e);
    }

  private:
    MixerSource with(const rb_effect& e) const {
        MixerSource m = *this;
        m.master_.push_back(e);
        return m;
    }
    static bool same(const std::vector<rb_effect>& a, const std::vector<rb_effect>& b) {
        return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * sizeof(rb_effect)) == 0);
    }
    void render() {
        Shared& s = *s_;
        if (!s.dirty && same(s.rendered_master, master_)) return;
        s.dirty = false;
        s.rendered_master = master_;
        s.rendered.clear(), s.active.clear();
        if (s.sources.empty()) return;
        std::vector<const Source*> ptrs;
        for (const Source& src : s.sources) ptrs.push_back(&src);
        detail::Flat flat(ptrs, s.starts);
        detail::Batch b(flat.descs, s.channels, s.rate, 0);
        flat.upload(b.h);
        if (!master_.empty()) check(rb_batch_set_master(b.h, master_.data(), (uint32_t)master_.size()), "rb_batch_set_master");
        uint64_t n = 0, w = 0;
        check(rb_batch_mix_len(b.h, &n), "rb_batch_mix_len");
        s.rendered.resize(n);
        check(rb_batch_render_mix(b.h, s.rendered.data(), n, &w), "rb_batch_render_mix");
        s.active.assign(n, 0);
        for (size_t i = 0; i < s.sources.size(); i++) {
            uint64_t len = 0;
            check(rb_batch_stream_out_len(b.h, i, &len), "rb_batch_stream_out_len");
            uint64_t st = (s.starts[i] + s.channels - 1) / s.channels * s.channels;
            for (uint64_t p = st; p < st + len && p < n; p++) s.active[p] = 1;
        }
    }
    std::shared_ptr<Shared> s_;
    std::vector<rb_effect> master_;
};

// mixer::mixer(channels, sample_rate) -> (Mixer, MixerSource) — src/mixer.rs:25-43
inline std::pair<Mixer, MixerSource> mixer(uint16_t channels, uint32_t sample_rate) {
    if (channels == 0 || sample_rate == 0) throw std::invalid_argument("channels / sample_rate are NonZero in rodio");
    auto s = std::make_shared<Shared>();
    s->channels = channels, s->rate = sample_rate;
    return {Mixer(s), MixerSource(s)};
}

// Streaming counterpart (rb_session_*): sources that arrive block by block -- decoders, capture -- behind one
// MixerSource-like pull.  `chains` describe the sources (channels, rate, adapters: .uniform(ch, rate)[.low_pass / .high_pass]
// [.amplify]); their PCM is pushed later.  next() hands out the mixer samples one at a time like Iterator::next
// (src/mixer.rs:120-136); std::nullopt while nothing can be rendered yet, `ended()` once every source is exhausted.
class LiveMixer {
  public:
    // mixer::mixer(channels, sample_rate) whose inputs arrive later: chains[i] ends in .uniform(channels, sample_rate)...
    // restarts: RB_SESSION_RESTARTS -- the mixer's conversion restarts where rodio's does, every min(span_len, 32768) samples of a
    // chain whose source reports a span, and behind take_duration.
    LiveMixer(const std::vector<Source>& chains, uint16_t channels, uint32_t sample_rate, uint32_t fifo_frames = 8192,
              uint32_t block_frames = 1024, bool restarts = false)
        : channels_(channels), rate_(sample_rate), block_frames_(block_frames) {
        std::vector<rb_stream_desc> descs;
        for (const Source& c : chains) descs.push_back(c.desc(0)), src_channels_.push_back(descs.back().channels);
        check(rb_session_create_ex(Context::get(), channels, sample_rate, descs.data(), descs.size(), fifo_frames, block_frames,
                                   restarts ? RB_SESSION_RESTARTS : 0u, &h_),
              "rb_session_create_ex");
    }
    LiveMixer(const LiveMixer&) = delete;
    LiveMixer& operator=(const LiveMixer&) = delete;
    ~LiveMixer() { rb_session_destroy(h_); }
    uint16_t channels() const { return channels_; }
    uint32_t sample_rate() const { return rate_; }
    // converter runs of source `i` that have produced an output so far (rb_session_source_runs)
    uint64_t source_runs(size_t i) const {
        uint64_t n = 0;
        check(rb_session_source_runs(h_, i, &n), "rb_session_source_runs");
        return n;
    }
    // more interleaved samples of source `i`; end_of_stream: its Iterator::next would return None after them
    void push(size_t i, const std::vector<Sample>& pcm, bool end_of_stream = false) {
        check(rb_session_push(h_, i, pcm.data(), pcm.size() / src_channels_.at(i), end_of_stream ? 1 : 0), "rb_session_push");
    }
    // The same with span marks (restarts only): after marks[k].at samples of this push the source reports marks[k].span_len
    // (0 = None) -- a decoder's packet lengths, as current_span_len() returns them (rb_session_push_spans).
    void push(size_t i, const std::vector<Sample>& pcm, const std::vector<rb_span_mark>& marks, bool end_of_stream = false) {
        check(rb_session_push_spans(h_, i, pcm.data(), pcm.size() / src_channels_.at(i), marks.data(), (uint32_t)marks.size(),
                                    end_of_stream ? 1 : 0), "rb_session_push_spans");
    }
    // Player::pause for n_frames frames: whole frames of 0.0 behind the source's push program, which is not pulled meanwhile
    void push_silence(size_t i, uint64_t n_frames) { check(rb_session_push_silence(h_, i, n_frames), "rb_session_push_silence"); }
    // Mixer::add (mixer.rs:58-66) for a source that was declared held (its desc().mix_start == RB_SESSION_HELD)
    void add(size_t i) { check(rb_session_start(h_, i), "rb_session_start"); }
    // queue a held source behind another one: Player::append / queue.rs:128-192
    void append_after(size_t i, size_t predecessor) { check(rb_session_follow(h_, i, predecessor), "rb_session_follow"); }
    void skip(size_t i) { check(rb_session_skip(h_, i), "rb_session_skip"); }   // Player::skip_one / stop
    // Amplify::set_factor on the chain's .amplify() (amplify.rs:25-29); Player::set_volume's Amplify sits before the resampler
    void set_amplify(size_t i, float factor) { check(rb_session_set_amplify(h_, i, factor), "rb_session_set_amplify"); }
    // Player::set_volume: the AMPLIFY in front of the mixer's conversion (src/player.rs:120-128, :180-186)
    void set_volume(size_t i, float factor) { check(rb_session_set_volume(h_, i, factor), "rb_session_set_volume"); }
    // mixer_source.amplify(a).limit(s).amplify(b) on the output (rb_session_set_master), before the first next()
    void set_master(const std::vector<rb_effect>& effects) {
        check(rb_session_set_master(h_, effects.data(), (uint32_t)effects.size()), "rb_session_set_master");
    }
    bool ended() const { return ended_ && at_ == block_.size(); }
    std::optional<Sample> next() {
        if (at_ == block_.size()) {
            if (ended_) return std::nullopt;
            block_.resize((size_t)block_frames_ * channels_);
            uint64_t written = 0;
            int e = 0;
            check(rb_session_render(h_, block_.data(), block_frames_, &written, &e), "rb_session_render");
            block_.resize((size_t)written * channels_);
            at_ = 0, ended_ = e != 0;
            if (block_.empty()) return std::nullopt;   // starved (or ended): nothing renderable right now
        }
        return block_[at_++];
    }

  private:
    rb_session* h_ = nullptr;
    uint16_t channels_;
    std::vector<uint16_t> src_channels_;   // the sources' own interleaving (a mono source in a stereo mixer pushes mono)
    uint32_t rate_, block_frames_;
    std::vector<Sample> block_;
    size_t at_ = 0;
    bool ended_ = false;
};

}  // namespace mixer

namespace conversions {
// SampleRateConverter::new(input, from, to, channels).collect() — src/conversions/sample_rate.rs:52-201
inline std::vector<Sample> SampleRateConverter(const std::vector<Sample>& input, uint32_t from, uint32_t to, uint16_t channels) {
    uint64_t n = 0;
    check(rb_sample_rate_out_len(input.size(), from, to, channels, &n), "rb_sample_rate_out_len");
    std::vector<Sample> out(n);
    check(rb_convert_sample_rate(Context::get(), input.data(), input.size(), from, to, channels, out.data(), n, &n),
          "rb_convert_sample_rate");
    out.resize(n);
    return out;
}
// ChannelCountConverter::new(input, from, to).collect() — src/conversions/channels.rs:28,:57-85
inline std::vector<Sample> ChannelCountConverter(const std::vector<Sample>& input, uint16_t from, uint16_t to) {
    uint64_t n = 0;
    check(rb_channels_out_len(input.size(), from, to, &n), "rb_channels_out_len");
    std::vector<Sample> out(n);
    check(rb_convert_channels(Context::get(), input.data(), input.size(), from, to, out.data(), n, &n), "rb_convert_channels");
    out.resize(n);
    return out;
}
}  // namespace conversions

}  // namespace rodio
