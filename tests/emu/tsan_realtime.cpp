// ThreadSanitizer driver for the emulated realtime.cu kernels (built by tests/test_realtime.py with -fsanitize=thread).
// rt_regrid's chunked neighbour scans are the only block barriers; they run over several chunks in both modes, with
// voiced frames inside, before and after each chunk.  rt_sola's per-warp results meet in shared memory.
#include <cmath>
#include <cstdio>
#include <vector>

#include "emu_realtime.cpp"

int main() {
    double s = 0;
    const int n_src = 700, n_dst = 600;
    std::vector<float> src(n_src), out(n_dst);
    for (int i = 0; i < n_src; ++i) src[i] = (i % 97 < 40 || i > 650) ? 0.f : 100.f + (float)(i % 13);
    std::vector<double> vsrc(n_src), vdst(n_dst);
    std::vector<int> prev(n_src);
    for (int mode : {0, 1}) {
        emu_rt_f0_regrid(src.data(), n_src, 0.01, 1.0, 1.25f, n_dst, mode ? 37 : 0, 512.0 / 44100.0, mode, 50.0, 1.5f,
                         out.data(), vsrc.data(), vdst.data(), prev.data());
        for (float v : out) s += v;
    }
    const int cf = 300, search = 70;
    std::vector<float> x(cf + search), buf(cf);
    for (int i = 0; i < cf + search; ++i) x[i] = std::sin(0.05f * (float)i);
    for (int i = 0; i < cf; ++i) buf[i] = std::sin(0.05f * (float)(i + 21));
    int shift = -1;
    emu_rt_sola(x.data(), buf.data(), cf, search, &shift);
    std::printf("done %g %d\n", s, shift);
    return 0;
}
