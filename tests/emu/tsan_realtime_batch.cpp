// ThreadSanitizer driver for the emulated batched realtime.cu entry points (built by tests/test_emu_realtime_batch.py
// with -fsanitize=thread).  Several rows each run rt_regrid's chunked neighbour scans (both modes, a row without voiced
// frames among them), rt_sola's per-warp results meet in shared memory per row, and the phase-vocoder crossfade reads
// each row's bins after their kernel.
#include <cmath>
#include <cstdio>
#include <vector>

#include "emu_realtime_batch.cpp"

int main() {
    double s = 0;
    const int rows = 3, n_src = 700, n_dst = 600;
    std::vector<float> src((size_t)rows * n_src), out((size_t)rows * n_dst), post{1.5f, 0.75f, 1.f};
    for (int r = 0; r < rows; ++r)
        for (int i = 0; i < n_src; ++i)
            src[(size_t)r * n_src + i] = (r == 2 || i % (97 - r) < 40 || i > 650) ? 0.f : 100.f + (float)(i % 13);
    std::vector<char> ws(rows * emu_rt_regrid_row_bytes(n_src, n_dst));
    for (int mode : {0, 1}) {
        emu_rt_f0_regrid_batch(src.data(), rows, n_src, 0.01, 1.0, 1.25f, n_dst, mode ? 37 : 0, 512.0 / 44100.0, mode,
                               50.0, post.data(), out.data(), ws.data());
        for (float v : out) s += v;
    }
    const int cf = 300, search = 70, block = 120;
    const long long stride = search + block + cf;
    std::vector<float> x(rows * stride), buf((size_t)rows * cf), fi(cf), fo(cf);
    for (int r = 0; r < rows; ++r) {
        for (int i = 0; i < stride; ++i) x[r * stride + i] = std::sin(0.05f * (float)(i + 3 * r));
        for (int i = 0; i < cf; ++i) buf[(size_t)r * cf + i] = std::sin(0.05f * (float)(i + 21 + r));
    }
    for (int i = 0; i < cf; ++i) {
        fi[i] = std::sin(0.5f * 3.14159265f * (float)i / (float)cf);
        fi[i] *= fi[i];
        fo[i] = 1.f - fi[i];
    }
    std::vector<int> shift(rows, -1);
    emu_rt_sola_batch(x.data(), stride, buf.data(), rows, cf, search, shift.data());
    std::vector<float> o((size_t)rows * block), nxt((size_t)rows * cf), bins((size_t)rows * 3 * (cf / 2 + 1));
    emu_rt_crossfade_batch(x.data(), stride, shift.data(), buf.data(), rows, fi.data(), fo.data(), block, cf, 1,
                           o.data(), nxt.data(), bins.data());
    for (float v : o) s += v;
    std::printf("done %g %d %d %d\n", s, shift[0], shift[1], shift[2]);
    return 0;
}
