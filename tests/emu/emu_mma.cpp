// One warp of host_emu.h's lane-collective mma_tf32 on raw per-lane fragments (built by tests/test_emu_mma.py, which
// lays them out from the PTX ISA's m16n8k8 tables itself).
#define B2D_HOST_EMU 1
#include "host_emu.h"

// a [32][4], b [32][2] (fp32 bit patterns as floats), d [32][4]: C in, D out
extern "C" int emu_mma_tf32(const float* a, const float* b, float* d) {
    emu::launch(1u, 1u, 32u, [&] {
        const int l = (int)threadIdx.x;
        uint32_t af[4];
        float df[4];
        for (int i = 0; i < 4; ++i) { af[i] = __float_as_uint(a[4 * l + i]); df[i] = d[4 * l + i]; }
        mma_tf32(df, af, __float_as_uint(b[2 * l]), __float_as_uint(b[2 * l + 1]));
        __syncwarp();                                   // every lane has read d before any writes it
        for (int i = 0; i < 4; ++i) d[4 * l + i] = df[i];
    });
    return 0;
}
