// frame_dev.cuh — warp-level device code shared by the 100 Hz kernels (frame_kernels.cu) and the analysis side (enc_kernels.cu):
// the reference's 320-point mixed-radix FFT butterflies (kiss_fft.c), lpc_from_cepstrum (freq.c:310-320) and the x86 float->int
// conversion of the (int)floor(...) sites.
#pragma once
#include <cstdint>
#include "engine.h"

namespace lpcnet_b200 {

// (int)v of a double as x86's cvttsd2si computes it: truncation toward zero, and INT_MIN (the "integer indefinite" value) for
// NaN and for anything outside int32.  CUDA's own conversion returns 0 for NaN and saturates out-of-range values, which the
// clamps after the reference's (int)floor(...) sites would turn into a different index.
__device__ __forceinline__ int cvtt_x86(double v)
{
    return (v > -2147483649.0 && v < 2147483648.0) ? (int)v : (int)0x80000000u;
}

struct c32 { float r, i; };
#define CMUL(m_, a_, b_) do { (m_).r = (a_).r * (b_).r - (a_).i * (b_).i; (m_).i = (a_).r * (b_).i + (a_).i * (b_).r; } while (0)
#define CADD(r_, a_, b_) do { (r_).r = (a_).r + (b_).r; (r_).i = (a_).i + (b_).i; } while (0)
#define CSUB(r_, a_, b_) do { (r_).r = (a_).r - (b_).r; (r_).i = (a_).i - (b_).i; } while (0)

// kiss_fft.c:101-170 (kf_bfly4), one butterfly; m == 1: the twiddle-free first stage
__device__ __forceinline__ void bfly4_first(c32 *Fout)
{
    c32 s0, s1;
    CSUB(s0, Fout[0], Fout[2]); CADD(Fout[0], Fout[0], Fout[2]);
    CADD(s1, Fout[1], Fout[3]); CSUB(Fout[2], Fout[0], s1); CADD(Fout[0], Fout[0], s1);
    CSUB(s1, Fout[1], Fout[3]);
    Fout[1].r = s0.r + s1.i; Fout[1].i = s0.i - s1.r;
    Fout[3].r = s0.r - s1.i; Fout[3].i = s0.i + s1.r;
}
__device__ __forceinline__ void bfly4(c32 *Fout, int m, const c32 t1, const c32 t2, const c32 t3)
{
    const int m2 = 2 * m, m3 = 3 * m;
    c32 s0, s1, s2, s3, s4, s5;
    CMUL(s0, Fout[m], t1); CMUL(s1, Fout[m2], t2); CMUL(s2, Fout[m3], t3);
    CSUB(s5, Fout[0], s1); CADD(Fout[0], Fout[0], s1);
    CADD(s3, s0, s2); CSUB(s4, s0, s2);
    CSUB(Fout[m2], Fout[0], s3);
    CADD(Fout[0], Fout[0], s3);
    Fout[m].r = s5.r + s4.i; Fout[m].i = s5.i - s4.r;
    Fout[m3].r = s5.r - s4.i; Fout[m3].i = s5.i + s4.r;
}
// kiss_fft.c:232-311 (kf_bfly5) with m = 64, N = 1, fstride = 1: butterfly u
__device__ __forceinline__ void bfly5_last(c32 *F0, int u, const c32 *__restrict__ tw)
{
    const int m = 64;
    const c32 ya = tw[m], yb = tw[2 * m];
    F0 += u;
    c32 *F1 = F0 + m, *F2 = F0 + 2 * m, *F3 = F0 + 3 * m, *F4 = F0 + 4 * m;
    c32 s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12;
    s0 = *F0;
    CMUL(s1, *F1, tw[u]); CMUL(s2, *F2, tw[2 * u]); CMUL(s3, *F3, tw[3 * u]); CMUL(s4, *F4, tw[4 * u]);
    CADD(s7, s1, s4); CSUB(s10, s1, s4); CADD(s8, s2, s3); CSUB(s9, s2, s3);
    F0->r = F0->r + (s7.r + s8.r); F0->i = F0->i + (s7.i + s8.i);
    s5.r = s0.r + (s7.r * ya.r + s8.r * yb.r); s5.i = s0.i + (s7.i * ya.r + s8.i * yb.r);
    s6.r = s10.i * ya.i + s9.i * yb.i; s6.i = -(s10.r * ya.i + s9.r * yb.i);
    CSUB(*F1, s5, s6); CADD(*F4, s5, s6);
    s11.r = s0.r + (s7.r * yb.r + s8.r * ya.r); s11.i = s0.i + (s7.i * yb.r + s8.i * ya.r);
    s12.r = s9.i * ya.i - s10.i * yb.i; s12.i = s10.r * yb.i - s9.r * ya.i;
    CADD(*F2, s11, s12); CSUB(*F3, s11, s12);
}


__device__ __constant__ short c_eband5ms[NB_BANDS] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 34, 40};               // freq.c:45-48
__device__ __constant__ float c_compensation[NB_BANDS] = {0.8f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 0.666667f, 0.5f, 0.5f, 0.5f,
                                                          0.333333f, 0.25f, 0.25f, 0.2f, 0.166667f, 0.173913f};                  // freq.c:50-52

// The four stages of opus_fft_impl for nfft = 320 (factors 5,4,4,4: lpcnet_tables.c:200) on data that is already scaled and
// digit-reversed in y[320] (shared memory), the butterflies of a stage dealt to `nthr` threads (thread `t`); `sync()` separates
// the stages (__syncwarp for a warp, __syncthreads for a block).
template <typename Sync>
__device__ __forceinline__ void fft320_stages(c32 *y, const c32 *__restrict__ tw, int t, int nthr, Sync sync)
{
    for (int i = t; i < 80; i += nthr) bfly4_first(y + 4 * i);                               // m = 1,  N = 80
    sync();
    for (int b = t; b < 80; b += nthr) { const int i = b >> 2, j = b & 3; bfly4(y + i * 16 + j, 4, tw[j * 20], tw[j * 40], tw[j * 60]); }      // m = 4,  N = 20, fstride 20
    sync();
    for (int b = t; b < 80; b += nthr) { const int i = b >> 4, j = b & 15; bfly4(y + i * 64 + j, 16, tw[j * 5], tw[j * 10], tw[j * 15]); }     // m = 16, N = 5,  fstride 5
    sync();
    for (int u = t; u < 64; u += nthr) bfly5_last(y, u, tw);
    sync();
}

// lpc_from_cepstrum (freq.c:310-320) by one warp: cep[18] (any memory) -> lpc[16] valid on lane 0.  y / Ex: shared scratch of the warp.
__device__ __forceinline__ void cepstrum_to_lpc_warp(const float *cep, c32 *y, float *Ex, const float *__restrict__ dct, const c32 *__restrict__ tw,
                                                     const int16_t *__restrict__ bitrev, float (&lpc)[LPC_ORDER], int lane)
{
    // idct (freq.c:230-240) + 10^x * compensation (freq.c:318): band i on lane i
    if (lane < NB_BANDS) {
        float sum = 0;
        for (int j = 0; j < NB_BANDS; j++) { const float t = j == 0 ? cep[0] + 4 : cep[j]; sum += t * __ldg(&dct[lane * NB_BANDS + j]); }
        const double idct_scale = sqrt(2. / NB_BANDS);
        const float e = (float)((double)sum * idct_scale);
        Ex[lane] = (float)(pow(10.0, (double)e) * (double)c_compensation[lane]);
    }
    __syncwarp();
    // interp_band_gain (freq.c:202-215) + Hermitian extension (freq.c:256-266) + scale & digit-reverse (kiss_fft.c:575-584)
    const float scale = 1.f / WINDOW_SIZE;
    for (int i = lane; i < WINDOW_SIZE; i += 32) {
        const int k = i < FREQ_SIZE ? i : WINDOW_SIZE - i;          // bin whose gain this sample carries
        float xr = 0.f;                                             // bin 160 stays 0 (freq.c:285)
        if (k < FREQ_SIZE - 1) {
            int b = 0;
            while (b < NB_BANDS - 2 && k >= c_eband5ms[b + 1] * 4) b++;
            const int band_size = (c_eband5ms[b + 1] - c_eband5ms[b]) * 4, j = k - c_eband5ms[b] * 4;
            const float frac = __fdiv_rn((float)j, (float)band_size);
            xr = (1 - frac) * Ex[b] + frac * Ex[b + 1];
        }
        const float xi = i < FREQ_SIZE ? 0.f : -0.f;
        const int o = bitrev[i];
        y[o].r = scale * xr; y[o].i = scale * xi;
    }
    __syncwarp();
    fft320_stages(y, tw, lane, 32, [] { __syncwarp(); });
    if (lane != 0) return;                                        // (the caller re-converges with __syncwarp / __syncthreads)
    float ac[LPC_ORDER + 1];
    ac[0] = WINDOW_SIZE * y[0].r;
    for (int i = 1; i < LPC_ORDER + 1; i++) ac[i] = WINDOW_SIZE * y[WINDOW_SIZE - i].r;
    ac[0] = (float)((double)ac[0] + ((double)ac[0] * 1e-4 + 320 / 12 / 38.));       // freq.c:292
    for (int i = 1; i < LPC_ORDER + 1; i++) ac[i] = (float)((double)ac[i] * (1 - 6e-5 * i * i));   // freq.c:294
#pragma unroll
    for (int i = 0; i < LPC_ORDER; i++) lpc[i] = 0;
    {                                                             // lpcn_lpc freq.c:86-127 (float build)
        float error = ac[0];
        if (ac[0] != 0) {
#pragma unroll
            for (int i = 0; i < LPC_ORDER; i++) {
                float rr = 0;
#pragma unroll
                for (int j = 0; j < i; j++) rr += lpc[j] * ac[i - j];
                rr += ac[i + 1];
                float r = __fdiv_rn(-rr, error);
                lpc[i] = r;
#pragma unroll
                for (int j = 0; j < (i + 1) >> 1; j++) {
                    float t1 = lpc[j], t2 = lpc[i - 1 - j];
                    lpc[j] = t1 + r * t2;
                    lpc[i - 1 - j] = t2 + r * t1;
                }
                error = error - (r * r) * error;
                if (error < .001f * ac[0]) break;
            }
        }
    }
}

}  // namespace lpcnet_b200
