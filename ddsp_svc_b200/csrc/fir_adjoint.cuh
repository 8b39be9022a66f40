// Device pieces of the direct-form adjoint of the time-varying FIR (ddsp/core.py:120-182) and of the impulse-response
// build (ddsp/core.py:254-270).  Each is a fixed-order fp32 / fp64 sum owned by one thread (block_scan: by one CTA), so
// no atomics.  block_scan and corr4 serve both the Sins backward (sins_bwd.cu) and the CombSub backward
// (combsub_bwd.cu); fir_t4 and irfft_adjoint_bin only the latter: sins_fir_bwd_kernel keeps its own inline copies,
// because calling either of them from there changes its register allocation (DESIGN §4.5b).
#pragma once

namespace b2d_firadj {

constexpr int kSub = 16;   // irfft adjoint: n = kSub a + r, exact table twiddles per (bin, r) and per a

// inclusive prefix (reverse = false) or suffix (reverse = true) sums of val[0, n) in fp64 into out, for a CTA of NT
// threads.  Thread t owns scan positions [t per, (t + 1) per); the chunk totals are combined by a
// Hillis-Steele scan in part[2 NT].  The summation order depends only on n.  Ends with a barrier.
template <int NT>
__device__ void block_scan(const float* val, double* out, int n, bool reverse, double* part) {
    const int tid = threadIdx.x;
    const int per = (n + NT - 1) / NT;
    double run = 0.0;
    for (int q = 0; q < per; ++q) {
        const int pos = tid * per + q;
        if (pos < n) {
            const int i = reverse ? n - 1 - pos : pos;
            run += (double)val[i];
            out[i] = run;
        }
    }
    part[tid] = run;
    __syncthreads();
    int src = 0;
    for (int off = 1; off < NT; off <<= 1) {
        double s = part[src * NT + tid];
        if (tid >= off) s += part[src * NT + tid - off];
        part[(1 - src) * NT + tid] = s;
        __syncthreads();
        src = 1 - src;
    }
    const double before = tid > 0 ? part[src * NT + tid - 1] : 0.0;
    for (int q = 0; q < per; ++q) {
        const int pos = tid * per + q;
        if (pos < n) out[reverse ? n - 1 - pos : pos] += before;
    }
    __syncthreads();
}

// Filter-gradient correlation of four taps 4 t4 .. 4 t4 + 3 (shared memory, 16-byte aligned):
//   acc[k] += sum_{i < 4 nq} v[i] g[4 t4 + k + i]
// with an 8-float register window sliding along g (one float4 of g and one of v per 16 FMAs).
__device__ __forceinline__ void corr4(const float* g, const float* v, int t4, int nq, float acc[4]) {
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* v4 = reinterpret_cast<const float4*>(v);
    float4 cur = g4[t4];
    for (int q = 0; q < nq; ++q) {
        const float4 nx = g4[q + t4 + 1];
        const float4 vv = v4[q];
        const float w[8] = {cur.x, cur.y, cur.z, cur.w, nx.x, nx.y, nx.z, nx.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            acc[k] = fmaf(vv.x, w[k], acc[k]);
            acc[k] = fmaf(vv.y, w[k + 1], acc[k]);
            acc[k] = fmaf(vv.z, w[k + 2], acc[k]);
            acc[k] = fmaf(vv.w, w[k + 3], acc[k]);
        }
        cur = nx;
    }
}

// Input-gradient pass of four samples 4 t4 .. 4 t4 + 3 through two filters hA, hB of 4 L4 taps (zero-padded):
//   a[k] += sum_tau hA[tau] g[4 t4 + k + tau],  c[k] += sum_tau hB[tau] g[4 t4 + k + tau]
__device__ __forceinline__ void fir_t4(const float* g, const float* hA, const float* hB, int t4, int L4, float a[4],
                                       float c[4]) {
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* hA4 = reinterpret_cast<const float4*>(hA);
    const float4* hB4 = reinterpret_cast<const float4*>(hB);
    float4 cur = g4[t4];
    for (int u = 0; u < L4; ++u) {
        const float4 nx = g4[t4 + u + 1];
        const float4 ha = hA4[u], hb = hB4[u];
        const float w[8] = {cur.x, cur.y, cur.z, cur.w, nx.x, nx.y, nx.z, nx.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            a[k] = fmaf(ha.x, w[k], a[k]);
            a[k] = fmaf(ha.y, w[k + 1], a[k]);
            a[k] = fmaf(ha.z, w[k + 2], a[k]);
            a[k] = fmaf(ha.w, w[k + 3], a[k]);
            c[k] = fmaf(hb.x, w[k], c[k]);
            c[k] = fmaf(hb.y, w[k + 1], c[k]);
            c[k] = fmaf(hb.z, w[k + 2], c[k]);
            c[k] = fmaf(hb.w, w[k + 3], c[k]);
        }
        cur = nx;
    }
}

// Adjoint of torch's c2r irfft (n = N = 2 (M - 1)) at bin j < M, from the un-rolled impulse-response gradient dr:
//   C_j = sum_n dr[n] cos(2 pi j n / N),  S_j = sum_n dr[n] sin(2 pi j n / N),
// with eo[n] = (dr[n] + dr[N-n], dr[n] - dr[N-n]) for 1 <= n < N/2 (zero up to kSub nblk), d0 = dr[0], dN = dr[N/2],
// cosT / sinT = cos / sin(2 pi t / N).  n = kSub a + r: cos / sin of (alpha_a + beta_r) from the exact table entries of
// alpha_a and beta_r.  Returns dH_j = (dre, dim): weight 2/N, and 1/N with the imaginary part dropped at DC and Nyquist.
__device__ __forceinline__ void irfft_adjoint_bin(int j, int M, int N, int nblk, const float* cosT, const float* sinT,
                                                  const float2* eo, float d0, float dN, float& dre, float& dim) {
    float cb[kSub], sb[kSub];
#pragma unroll
    for (int r = 0; r < kSub; ++r) {
        const int idx = (j * r) % N;
        cb[r] = cosT[idx];
        sb[r] = sinT[idx];
    }
    float C = 0.f, S = 0.f;
    int ia = 0;
    const int step = (j * kSub) % N;
    for (int a = 0; a < nblk; ++a) {
        float U = 0.f, V = 0.f, U2 = 0.f, V2 = 0.f;
#pragma unroll
        for (int r = 0; r < kSub; ++r) {
            const float2 e = eo[a * kSub + r];
            U = fmaf(e.x, cb[r], U);
            V = fmaf(e.x, sb[r], V);
            U2 = fmaf(e.y, cb[r], U2);
            V2 = fmaf(e.y, sb[r], V2);
        }
        const float ca = cosT[ia], sa = sinT[ia];
        C = fmaf(ca, U, fmaf(-sa, V, C));          // sum e cos(alpha + beta)
        S = fmaf(sa, U2, fmaf(ca, V2, S));         // sum o sin(alpha + beta)
        ia += step;
        if (ia >= N) ia -= N;
    }
    C += d0 + ((j & 1) ? -dN : dN);
    const bool edge = (j == 0 || j == M - 1);
    const float wj = (edge ? 1.0f : 2.0f) / (float)N;
    dre = wj * C;
    dim = edge ? 0.f : -wj * S;
}

}  // namespace b2d_firadj
