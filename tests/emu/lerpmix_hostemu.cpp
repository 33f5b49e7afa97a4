// librodio_b200_hostemu_lerpmix.so (test infrastructure): librodio_b200_hostemu.so (hostemu.cpp, included below unchanged) with
// k_lerp_mix emulated as the kernel runs it, and with the exact-order batches that the planner gives k_lerp_mix (rb_fused.cu)
// planned as well.  hostemu.cpp's own definitions of the two entry points are renamed on the way in and are not used here.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>

#define rb_lerpmix_launch hostemu_lerpmix_loop
#define rb_fused_try_create hostemu_fused_try_create
#include "hostemu.cpp"
#undef rb_lerpmix_launch
#undef rb_fused_try_create

cudaError_t rb_lerpmix_launch(const rb_lerpmix_args& a, cudaStream_t st);
cudaError_t rb_fused_try_create(const rb_fused_stream* streams, size_t n_streams, uint16_t mixer_channels, float* d_out, uint64_t mix_len,
                                uint32_t flags, int sm_count, cudaStream_t st, rb_fused_plan** out);

// ---- k_lerp_mix (rb_lanes.cu): every CTA (tile, group) walked as the kernel walks it -- descriptor chunks of LM_GROUP rows, stages
// of LM_ROWS rows whose windows are copied into LM_STAGES rotating buffers two stages ahead of the sums, window rows with the
// exact-reciprocal step, global rows with the IEEE division, the partial last tile, the write rule -- in the kernel's expressions.
// Position k of the tile stands for thread k % 256, u = k / 256.  Every input read is checked against the row's input rounded out
// to 16-byte granules (what a cp.async or an __ldg may touch): a read outside it aborts, naming row and tile.
namespace lm {
constexpr int U = 4, ROWS = 4, STAGES = 3, GROUP = 64, WQ = 260, TILE = 256 * U;
constexpr uint32_t GLOBAL = 0xffffffffu;
void check_read(const rb_lerpmix_args& a, uint32_t r, uintptr_t s, uint64_t n_floats, uint64_t tile, uint32_t g, const char* what) {
    const rb_lerpmix_row& row = a.rows[r];
    const lanes::Row& lr = a.lane_rows[row.row];
    const uintptr_t in = reinterpret_cast<uintptr_t>(lr.in);
    const uintptr_t lo = in & ~(uintptr_t)15, hi = (in + lr.L * sizeof(float) + 15) & ~(uintptr_t)15;
    const uintptr_t e = s + n_floats * sizeof(float);
    if (s >= lo && e <= hi && e >= s) return;
    fprintf(stderr, "k_lerp_mix: out-of-range read: %s of row %u (stream %u, %llu input frames) on tile %llu of group %u reads floats "
            "[%lld, %lld) of its input\n", what, r, row.row, (unsigned long long)lr.L, (unsigned long long)tile, g,
            (long long)(intptr_t)(s - in) / 4, (long long)(intptr_t)(e - in) / 4);
    fflush(stderr);
    abort();
}
float load(uintptr_t addr) {
    float v;
    std::memcpy(&v, reinterpret_cast<const void*>(addr), sizeof v);
    return v;
}
}  // namespace lm

cudaError_t rb_lerpmix_launch(const rb_lerpmix_args& a, cudaStream_t) {
    using namespace lm;
    std::vector<float> win((size_t)STAGES * ROWS * WQ * 4);
    std::vector<uint32_t> tap(TILE), pos(TILE);
    std::vector<float> numf(TILE), acc(TILE);
    std::vector<char> any(TILE);
    const uint64_t n_tiles = (a.mix_len + TILE - 1) / TILE;
    for (uint32_t g = 0; g < a.n_groups; g++)
        for (uint64_t bx = 0; bx < n_tiles; bx++) {
            const uint64_t tile_lo = bx * TILE;
            const uint64_t tile_hi = std::min<uint64_t>(a.mix_len, tile_lo + TILE);
            const uint32_t r_lo = g * a.rows_per_group, r_hi = std::min(a.n_rows, r_lo + a.rows_per_group);
            const uint64_t base = std::max(tile_lo, a.origin);
            const uint64_t i_tile = ((base - a.origin) * (uint64_t)a.from) / a.to;
            const uint32_t n_win = (uint32_t)((((std::max(tile_hi - 1, base) - a.origin) * (uint64_t)a.from) / a.to) - i_tile) + 2;
            for (int k = 0; k < TILE; k++) {
                const uint64_t n = tile_lo + k;
                const uint64_t prod = (std::max(n, base) - a.origin) * (uint64_t)a.from;
                const uint64_t i = prod / a.to;
                tap[k] = (uint32_t)(i - i_tile), numf[k] = (float)(uint32_t)(prod - i * a.to), pos[k] = (uint32_t)n;
                acc[k] = 0.0f, any[k] = 0;
            }
            const float den = a.den_f, rcp = a.rcp_den;
            const uint32_t t_lo = (uint32_t)tile_lo, t_hi = (uint32_t)tile_hi;
            const bool win_ok = n_win + 3 <= WQ * 4;
            const bool full_tile = tile_hi - tile_lo == TILE;
            bool any_win = false;
            for (uint32_t rs = r_lo; rs < r_hi; rs += GROUP) {
                const uint32_t n_st = std::min((uint32_t)GROUP, r_hi - rs);
                uint32_t woff[GROUP];
                for (uint32_t t = 0; t < n_st; t++) {
                    const rb_lerpmix_row& row = a.rows[rs + t];
                    const bool unsafe = (a.lane_rows[row.row].flags & lanes::ROW_UNSAFE) != 0;
                    const bool w_ok = win_ok && !unsafe && row.lo <= t_lo && row.hi_int >= t_hi;
                    const uint32_t off = (uint32_t)(((reinterpret_cast<uintptr_t>(row.p) + i_tile * sizeof(float)) >> 2) & 3u);
                    woff[t] = w_ok ? (t % ROWS) * (WQ * 4) + off : GLOBAL;
                }
                const uint32_t n_stages = (n_st + ROWS - 1) / ROWS;
                std::fill(win.begin(), win.end(), std::numeric_limits<float>::quiet_NaN());   // shared memory holds no zeros
                auto issue = [&](uint32_t stage) {          // the window copies of a stage, 16-byte quads
                    for (uint32_t jrow = 0; jrow < ROWS; jrow++) {
                        const uint32_t r = stage * ROWS + jrow;
                        if (stage >= n_stages || r >= n_st || woff[r] == GLOBAL) continue;
                        const uint32_t off = woff[r] & 3u;
                        const uintptr_t src = reinterpret_cast<uintptr_t>(a.rows[rs + r].p) + (i_tile - off) * sizeof(float);
                        float* dst = win.data() + ((size_t)(stage % STAGES) * ROWS + jrow) * WQ * 4;
                        const uint32_t nq = (off + n_win + 3) >> 2;
                        if (nq > (uint32_t)WQ) {
                            fprintf(stderr, "k_lerp_mix: window of row %u on tile %llu of group %u overflows its buffer\n", rs + r, (unsigned long long)bx, g);
                            abort();
                        }
                        check_read(a, rs + r, src, 4ull * nq, bx, g, "window copy");
                        std::memcpy(dst, reinterpret_cast<const void*>(src), (size_t)nq * 16);
                    }
                };
                issue(0);
                issue(1);
                for (uint32_t stage = 0; stage < n_stages; stage++) {
                    issue(stage + 2);                       // into the buffer of stage - 1, which is no longer read
                    const float* buf = win.data() + (size_t)(stage % STAGES) * ROWS * WQ * 4;
                    const uint32_t j_hi = std::min((uint32_t)ROWS, n_st - stage * ROWS);
                    for (uint32_t j = 0; j < j_hi; j++) {
                        const uint32_t r = stage * ROWS + j;
                        const rb_lerpmix_row& row = a.rows[rs + r];
                        if (woff[r] != GLOBAL) {
                            const float* w = buf + woff[r];
                            for (int k = 0; k < TILE; k++) {
                                const float xa = w[tap[k]], xb = w[tap[k] + 1];
                                const float m = (xb - xa) * numf[k];
                                const float q0 = m * rcp;
                                const float q = std::fmaf(std::fmaf(-q0, den, m), rcp, q0);
                                float x = xa + q;
                                if (a.has_post) x = x * row.post;
                                if (full_tile || pos[k] < t_hi) acc[k] = acc[k] + x;
                            }
                            any_win = true;
                            continue;
                        }
                        if (row.hi <= t_lo || row.lo >= t_hi) continue;
                        const uintptr_t p = reinterpret_cast<uintptr_t>(row.p) + i_tile * sizeof(float);
                        for (int k = 0; k < TILE; k++) {
                            if (pos[k] < row.lo || pos[k] >= row.hi || pos[k] >= t_hi) continue;
                            const uintptr_t pa = p + (uint64_t)tap[k] * sizeof(float);
                            check_read(a, rs + r, pa, 1, bx, g, "left tap");
                            const float xa = load(pa);
                            float x = xa;
                            if (pos[k] < row.hi_int) {
                                check_read(a, rs + r, pa + sizeof(float), 1, bx, g, "right tap");
                                x = xa + ((load(pa + sizeof(float)) - xa) * numf[k]) / den;
                            }
                            if (a.has_post) x = x * row.post;
                            acc[k] = acc[k] + x, any[k] = 1;
                        }
                    }
                }
            }
            float* out = a.out + (uint64_t)g * a.pstride;
            for (int k = 0; k < TILE; k++)
                if (pos[k] < t_hi && (any[k] || any_win || a.n_groups == 1)) out[pos[k]] = acc[k];
        }
    return cudaSuccess;
}

// RB_MIX_EXACT_ORDER: filter-free mono chains below 1024 streams are k_lerp_mix's, in one group (rb_fused.cu); every other
// exact-order batch takes a kernel that has no emulation here.  Other batches are planned as hostemu.cpp plans them.
cudaError_t rb_fused_try_create(const rb_fused_stream* streams, size_t n_streams, uint16_t mixer_channels, float* d_out, uint64_t mix_len,
                                uint32_t flags, int sm_count, cudaStream_t st, rb_fused_plan** out) {
    *out = nullptr;
    if (!(flags & RB_MIX_EXACT_ORDER))
        return hostemu_fused_try_create(streams, n_streams, mixer_channels, d_out, mix_len, flags, sm_count, st, out);
    if (n_streams == 0 || n_streams >= 1024 || mix_len == 0) return cudaSuccess;
    std::vector<FusedRow> rows(n_streams);
    uint32_t n_pre = 0, n_mid = 0, n_post = 0, has_u = 0, has_b = 0, front = 0;
    bool mixed_u = false, all_f32 = true;
    if (!fused_parse_rows(streams, n_streams, mixer_channels, rows, n_pre, n_mid, n_post, has_u, has_b, mixed_u, front)) return cudaSuccess;
    if (has_b || front || !has_u || mixer_channels != 1 || (flags & (RB_FUSED_LANES | RB_FUSED_DUO))) return cudaSuccess;
    for (size_t i = 0; i < n_streams; i++) all_f32 = all_f32 && streams[i].fmt == RB_FMT_F32;
    rb_lanes_plan* lanes = nullptr;
    cudaError_t e = fused_lanes_hook(rows, n_streams, mixer_channels, all_f32, n_pre, n_mid, n_post, has_u, has_b, front, flags, sm_count, d_out,
                                     mix_len, st, &lanes);
    if (e != cudaSuccess || !lanes) return e;
    if (rb_lanes_kind(lanes) != 6) {   // only k_lerp_mix keeps the sequential order
        rb_lanes_destroy(lanes);
        return cudaSuccess;
    }
    *out = new rb_fused_plan{lanes};
    return cudaSuccess;
}
