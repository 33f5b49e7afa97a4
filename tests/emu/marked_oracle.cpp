// marked_oracle.cpp — test infrastructure: the CPU oracle (oracle/rodio_oracle_capi.cpp, compiled into this unit unchanged) with a
// base source whose current_span_len() follows a mark table.  rodio's symphonia decoder reports the length of the packet it
// decoded last (src/decoder/symphonia.rs:199-201: the first packet is decoded in the constructor, :173-179, the next one by the
// next() that finds the buffer exhausted, :344-411); the oracle's literal UniformSourceIterator asks at every bootstrap before it
// pulls (src/source/uniform.rs:50-68).  Loaded with ctypes by tests/emu/marked_oracle.py; never linked into the product library.
#include "../../oracle/rodio_oracle_capi.cpp"

namespace {
// Vec-backed: `span` before the first mark, then marks[k].second once marks[k].first samples have been yielded (0 = None).
struct MarkedSource : Source {
    std::shared_ptr<const std::vector<Sample>> data;
    std::shared_ptr<const std::vector<std::pair<uint64_t, uint64_t>>> marks;
    size_t pos = 0, k = 0;
    uint16_t ch;
    uint32_t rate;
    std::optional<size_t> span;
    MarkedSource(uint16_t c, uint32_t r, std::shared_ptr<const std::vector<Sample>> d, std::optional<size_t> s,
                 std::shared_ptr<const std::vector<std::pair<uint64_t, uint64_t>>> m)
        : data(std::move(d)), marks(std::move(m)), ch(c), rate(r), span(s) {
        follow();
    }
    void follow() {
        for (; k < marks->size() && (*marks)[k].first <= pos; k++)
            span = (*marks)[k].second ? std::optional<size_t>((size_t)(*marks)[k].second) : std::nullopt;
    }
    std::optional<Sample> next() override {
        if (pos >= data->size()) return std::nullopt;
        Sample v = (*data)[pos++];
        follow();
        return v;
    }
    std::optional<size_t> current_span_len() const override { return span; }
    uint16_t channels() const override { return ch; }
    uint32_t sample_rate() const override { return rate; }
    Src clone() const override { return std::make_unique<MarkedSource>(*this); }
};

// The stream's chain over a MarkedSource of its PCM (span_len: the report before the first mark); `marks`: n pairs (samples
// yielded, span_len) in increasing order
Src build_marked(const ro_stream& s, const uint64_t* marks, uint64_t n) {
    auto table = std::make_shared<std::vector<std::pair<uint64_t, uint64_t>>>();
    for (uint64_t k = 0; k < n; k++) table->push_back({marks[2 * k], marks[2 * k + 1]});
    auto data = std::make_shared<const std::vector<Sample>>(s.pcm, s.pcm + s.n_samples);
    std::optional<size_t> span;
    if (s.span_len) span = (size_t)s.span_len;
    return apply_effects(std::make_unique<MarkedSource>(s.channels, s.sample_rate, data, span, std::move(table)), s.effects, s.n_effects);
}
}  // namespace

extern "C" {
// ro_chain_uniform with the stream's PCM a MarkedSource
int ro_marked_chain_uniform(const ro_stream* s, const uint64_t* marks, uint64_t n_marks, uint16_t mixer_ch, uint32_t mixer_rate, float* out,
                            uint64_t cap, uint64_t* n_out) {
    Src src = build_marked(*s, marks, n_marks);
    if (!src) return 1;
    UniformSourceIterator u(std::move(src), mixer_ch, mixer_rate);
    return drain(u, out, cap, n_out);
}
// ro_mixer with every stream's PCM a MarkedSource: stream i follows marks[2 * first[i] .. 2 * first[i + 1])
int ro_marked_mixer(const ro_stream* streams, uint64_t n_streams, const uint64_t* first, const uint64_t* marks, uint16_t ch, uint32_t rate,
                    float* out, uint64_t cap, uint64_t* n_out) {
    MixerSource mx(ch, rate);
    std::vector<uint64_t> order(n_streams);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return streams[a].mix_start < streams[b].mix_start; });
    uint64_t next_add = 0, pos = 0;
    while (true) {
        while (next_add < n_streams && streams[order[next_add]].mix_start <= pos) {
            const uint64_t i = order[next_add];
            Src s = build_marked(streams[i], marks + 2 * first[i], first[i + 1] - first[i]);
            if (!s) return 1;
            mx.add(std::move(s));
            next_add++;
        }
        auto v = mx.next();
        if (!v) {
            if (next_add >= n_streams && mx.still_pending.empty()) break;
            if (pos < cap) out[pos] = 0.0f;   // a gap: written as 0.0, as ro_mixer does
        } else if (pos < cap)
            out[pos] = *v;
        pos++;
    }
    *n_out = pos;
    return pos <= cap ? 0 : 8;
}
}
