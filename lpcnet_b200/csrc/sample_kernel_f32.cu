// sample_kernel_f32.cu — per-sample loop for the FLOAT flavour of the model (reference built with
// --disable-dot-product / -DDISABLE_DOT_PROD: pinned oracle build "B"; BASELINE config 2 "fp16 weights").
//
// Same mapping as the int8 kernel (one CTA = 32 streams, lane == stream, 16 compute warps + 1 sampler warp) but the
// arithmetic of the recurrent layers is fp32 and ORDER-SENSITIVE, so the structure is simpler and slower:
//   * sparse_sgemv_accum8x4 float (src/vec_avx.h:865-903): every output row is a sequential FMA chain that starts
//     from bias + diag*h (+ gathered input term) and walks the blocks in idx order, inputs c = 0..3 inside a block.
//     A lane that owns the row reproduces it exactly with __fmaf_rn; the chain cannot be split or pre-computed.
//   * sgemv_accum16 (src/vec_avx.h:618-643) for the GRU_B recurrent part: y = fma(W[j*48+i], hB[j], y), j ascending.
//   * compute_sparse_gru / compute_gruB use `bias`, not `subias` (USE_SU_BIAS is only defined with DOT_PROD,
//     src/vec_avx.h:39-41, src/nnet.c:346-360,425-430).
// Weights sit in shared memory as fp16 (64 B per 8x4 block, [4 in][8 out]); the loader only accepts blobs whose
// float weights are exactly representable, so results equal the fp32 reference bit for bit.  The GRU_A state tile is
// fp32 [384][32].  The GRU_A input term is gathered per lane (no transposition tile: shared memory is full).
#include <cstdint>
#include <cuda_fp16.h>
#ifndef LPCNET_NA
#define LPCNET_NA 384          // GRU_A units this translation unit is compiled for
#endif
#include "sample_common.cuh"

namespace lpcnet_b200 {
namespace LPCNET_KNS {

namespace {

constexpr int F_THREADS = (F_NWC + 1) * 32;

enum { FB_IDX = 1, FB_READ = 2, FB_X = 3, FB_ACCB = 4, FB_HB = 5 };

// 8 gathered conditioning inputs of one (gate, neuron group) for this lane's stream: ((cond + E_sig[a]) + E_pred[b]) + E_exc[c]
__device__ __forceinline__ void gather8(float g[8], const float *__restrict__ c, const float *__restrict__ e0,
                                        const float *__restrict__ e1, const float *__restrict__ e2, int off)
{
    const float4 c0 = ldg4(c + off), c1 = ldg4(c + off + 4), s0 = ldg4(e0 + off), s1 = ldg4(e0 + off + 4);
    const float4 p0 = ldg4(e1 + off), p1 = ldg4(e1 + off + 4), x0 = ldg4(e2 + off), x1 = ldg4(e2 + off + 4);
    g[0] = __fadd_rn(__fadd_rn(__fadd_rn(c0.x, s0.x), p0.x), x0.x); g[1] = __fadd_rn(__fadd_rn(__fadd_rn(c0.y, s0.y), p0.y), x0.y);
    g[2] = __fadd_rn(__fadd_rn(__fadd_rn(c0.z, s0.z), p0.z), x0.z); g[3] = __fadd_rn(__fadd_rn(__fadd_rn(c0.w, s0.w), p0.w), x0.w);
    g[4] = __fadd_rn(__fadd_rn(__fadd_rn(c1.x, s1.x), p1.x), x1.x); g[5] = __fadd_rn(__fadd_rn(__fadd_rn(c1.y, s1.y), p1.y), x1.y);
    g[6] = __fadd_rn(__fadd_rn(__fadd_rn(c1.z, s1.z), p1.z), x1.z); g[7] = __fadd_rn(__fadd_rn(__fadd_rn(c1.w, s1.w), p1.w), x1.w);
}

// y[r] = fma(w[c][r], x[pos+c], y[r]) for the blocks of one row group, in list order (sparse_sgemv_accum8x4, float)
__device__ __forceinline__ void gemv_f32(float y[8], const uint8_t *__restrict__ w, const uint16_t *__restrict__ meta, int nb,
                                         const uint8_t *__restrict__ xs_lane)
{
    for (int b = 0; b < nb; b++) {
        const uint8_t *xr = xs_lane + meta[b];                   // row `pos` of the [384][32] fp32 state tile, this lane's column
        const float x[4] = {*reinterpret_cast<const float *>(xr), *reinterpret_cast<const float *>(xr + 128),
                            *reinterpret_cast<const float *>(xr + 256), *reinterpret_cast<const float *>(xr + 384)};
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const uint4 raw = *reinterpret_cast<const uint4 *>(w + c * 16);          // 8 halves = w[c][0..7]
            const __half2 *h2 = reinterpret_cast<const __half2 *>(&raw);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const float2 f = __half22float2(h2[k]);
                y[2 * k] = __fmaf_rn(f.x, x[c], y[2 * k]);
                y[2 * k + 1] = __fmaf_rn(f.y, x[c], y[2 * k + 1]);
            }
        }
        w += 64;
    }
}

}  // namespace

// The body of the kernel for the streams of `P` that CTA `cta` of their batch holds.  A single-batch launch runs it with its own
// parameters and blockIdx.x; a group launch with the parameters of the CTA's member and the member-local CTA index.
__device__ __forceinline__ void sample_body_f32(const SampleParams &P, int cta)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const SmemLayout &L = P.L;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = P.n_streams;
    const int s_raw = cta * P.spc + lane;                        // lanes >= spc are dead slots (shadow the last stream, stores masked)
    const bool live = lane < P.spc && s_raw < n;
    const int s = live ? s_raw : n - 1;

    const uint32_t bar = smem_u32(smem + F_MBAR);
    if (threadIdx.x == 0) { mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    if (threadIdx.x == 0) stage_image(smem_u32(smem + F_IMAGE), P.image, L.image_bytes, bar);
    const uint16_t *rcp = reinterpret_cast<const uint16_t *>(smem + F_IMAGE + FI_RCP);
    float *xs = reinterpret_cast<float *>(smem + F_XS);
    float *hBs = reinterpret_cast<float *>(smem + F_HB);          // [2][16][32]
    float *accB = reinterpret_cast<float *>(smem + F_ACCB);
    int *idx_s = reinterpret_cast<int *>(smem + F_IDX);
    const int spf = P.spf;
    mbar_wait(bar, 0);

    if (warp < F_NWC) {
        const uint32_t *grpA = reinterpret_cast<const uint32_t *>(smem + F_IMAGE + FI_GRPA);
        const uint32_t *dirA = reinterpret_cast<const uint32_t *>(smem + F_IMAGE + FI_DIRA) + warp * F_GPW * 3 * 2;
        const float *parA = reinterpret_cast<const float *>(smem + F_IMAGE + FI_PARA) + warp * F_GPW * 3 * 16;
        const uint16_t *metaA = reinterpret_cast<const uint16_t *>(smem + L.metaA);
        const uint8_t *wA = smem + L.wA;
        const uint32_t *dirB = reinterpret_cast<const uint32_t *>(smem + F_IMAGE + FI_DIRB);
        const uint16_t *metaB = reinterpret_cast<const uint16_t *>(smem + L.metaB);
        const uint8_t *wB = smem + L.wB;
        const float *parB = reinterpret_cast<const float *>(smem + F_IMAGE + FI_PARB);
        const float *wBrec = reinterpret_cast<const float *>(smem + L.wBrecF);
        const uint8_t *xs_lane = reinterpret_cast<const uint8_t *>(xs) + lane * 4;

        int grp[F_GPW];
        float h[F_GPW][8];
#pragma unroll
        for (int sl = 0; sl < F_GPW; sl++) {
            grp[sl] = (int)grpA[warp * F_GPW + sl];
#pragma unroll
            for (int i = 0; i < 8; i++) { h[sl][i] = P.hA[(size_t)(8 * grp[sl] + i) * n + s]; xs[(8 * grp[sl] + i) * 32 + lane] = h[sl][i]; }
        }
        const int jb = warp;                                       // GRU_B neuron finished by this warp
        float hb = P.hB[(size_t)jb * n + s];
        hBs[jb * 32 + lane] = hb;
        bar_sync(FB_X, F_NWC * 32);

        int step = 0;
        for (int f = 0; f < P.nframes; f++) {
            const float *condA = P.condA + ((size_t)f * n + s) * (3 * NA);
            const float *condBp = P.condB + ((size_t)f * n + s) * (3 * NB);
            for (int t = 0; t < spf; t++, step++) {
                const int cur = step & 1, nxt = cur ^ 1;
                bar_sync(FB_IDX, F_THREADS);
                const float *e_sig = P.emb_sig + (size_t)idx_s[lane] * (3 * NA);
                const float *e_pred = P.emb_pred + (size_t)idx_s[32 + lane] * (3 * NA);
                const float *e_exc = P.emb_exc + (size_t)idx_s[64 + lane] * (3 * NA);
#pragma unroll
                for (int sl = 0; sl < F_GPW; sl++) {
                    const int g = grp[sl];
                    const float *par = parA + sl * 3 * 16;
                    const uint32_t *dir = dirA + sl * 3 * 2;
                    float gin[8], y[8], r[8];
                    // reset gate (nnet.c:431-435): chain starts from bias + diag*h + gin
                    gather8(gin, condA, e_sig, e_pred, e_exc, NA + 8 * g);
#pragma unroll
                    for (int i = 0; i < 8; i++) y[i] = __fadd_rn(__fadd_rn(par[16 + i], __fmul_rn(par[24 + i], h[sl][i])), gin[i]);
                    gemv_f32(y, wA + (size_t)dir[2] * 64, metaA + dir[2], (int)dir[3], xs_lane);
#pragma unroll
                    for (int i = 0; i < 8; i++) r[i] = sigmoid_approx(y[i], rcp);
                    // candidate (nnet.c:436-445)
                    gather8(gin, condA, e_sig, e_pred, e_exc, 2 * NA + 8 * g);
#pragma unroll
                    for (int i = 0; i < 8; i++) y[i] = __fadd_rn(par[32 + i], __fmul_rn(par[40 + i], h[sl][i]));
                    gemv_f32(y, wA + (size_t)dir[4] * 64, metaA + dir[4], (int)dir[5], xs_lane);
#pragma unroll
                    for (int i = 0; i < 8; i++) r[i] = tanh_approx(__fadd_rn(__fmul_rn(y[i], r[i]), gin[i]), rcp);     // r now holds h~
                    // update gate and new state (nnet.c:446-447)
                    gather8(gin, condA, e_sig, e_pred, e_exc, 8 * g);
#pragma unroll
                    for (int i = 0; i < 8; i++) y[i] = __fadd_rn(__fadd_rn(par[i], __fmul_rn(par[8 + i], h[sl][i])), gin[i]);
                    gemv_f32(y, wA + (size_t)dir[0] * 64, metaA + dir[0], (int)dir[1], xs_lane);
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const float z = sigmoid_approx(y[i], rcp);
                        h[sl][i] = __fadd_rn(__fmul_rn(z, h[sl][i]), __fmul_rn(__fsub_rn(1.f, z), r[i]));
                    }
                }
                bar_sync(FB_READ, F_NWC * 32);                          // every warp has finished reading the old state tile
#pragma unroll
                for (int sl = 0; sl < F_GPW; sl++)
#pragma unroll
                    for (int i = 0; i < 8; i++) xs[(8 * grp[sl] + i) * 32 + lane] = h[sl][i];
                bar_sync(FB_X, F_NWC * 32);
                // GRU_B input side (nnet.c:346-352): row group `warp` (6 warps), full chain in idx order
                if (warp < 6) {
                    float y[8];
                    const float4 c0 = ldg4(condBp + warp * 8), c1 = ldg4(condBp + warp * 8 + 4);
                    const float cb[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
                    for (int i = 0; i < 8; i++) y[i] = __fadd_rn(parB[warp * 8 + i], cb[i]);
                    const uint32_t b0 = dirB[(warp * F_KPARTS) * 2], nb = dirB[(warp * F_KPARTS) * 2 + 1];
                    gemv_f32(y, wB + (size_t)b0 * 64, metaB + b0, (int)nb, xs_lane);
#pragma unroll
                    for (int i = 0; i < 8; i++) accB[(warp * 8 + i) * 32 + lane] = y[i];
                }
                bar_sync(FB_ACCB, F_NWC * 32);
                {   // GRU_B finish for neuron jb: recurrent chains (sgemv_accum16), gates (nnet.c:353-371)
                    const float *hbo = hBs + cur * NB * 32;
                    float rz = parB[3 * NB + jb], rr = parB[4 * NB + jb], rh = parB[5 * NB + jb];
#pragma unroll
                    for (int j = 0; j < NB; j++) {
                        const float xj = hbo[j * 32 + lane];
                        rz = __fmaf_rn(wBrec[j * 3 * NB + jb], xj, rz);
                        rr = __fmaf_rn(wBrec[j * 3 * NB + NB + jb], xj, rr);
                        rh = __fmaf_rn(wBrec[j * 3 * NB + 2 * NB + jb], xj, rh);
                    }
                    const float zz = sigmoid_approx(__fadd_rn(accB[jb * 32 + lane], rz), rcp);
                    const float rrr = sigmoid_approx(__fadd_rn(accB[(NB + jb) * 32 + lane], rr), rcp);
                    const float hh = tanh_approx(__fadd_rn(accB[(2 * NB + jb) * 32 + lane], __fmul_rn(rh, rrr)), rcp);
                    hb = __fadd_rn(__fmul_rn(zz, hb), __fmul_rn(__fsub_rn(1.f, zz), hh));
                    hBs[nxt * NB * 32 + jb * 32 + lane] = hb;
                }
                __threadfence_block();
                bar_arrive(FB_HB, F_THREADS);
            }
        }
        if (live) {
#pragma unroll
            for (int sl = 0; sl < F_GPW; sl++)
#pragma unroll
                for (int i = 0; i < 8; i++) P.hA[(size_t)(8 * grp[sl] + i) * n + s] = h[sl][i];
            P.hB[(size_t)jb * n + s] = hb;
        }
    } else {
        // ----------------------------------------------------------------- sampler warp (identical arithmetic to the int8 kernel)
        const float *logit = reinterpret_cast<const float *>(smem + F_IMAGE + FI_LOGIT);
        const float *u2l = reinterpret_cast<const float *>(smem + F_IMAGE + FI_U2L);
        const float *fcb = reinterpret_cast<const float *>(smem + F_IMAGE + FI_FCB);
        const float *fcf = reinterpret_cast<const float *>(smem + F_IMAGE + FI_FCF);
        float ls[LPC_ORDER], lpc[LPC_ORDER];
#pragma unroll
        for (int j = 0; j < LPC_ORDER; j++) ls[j] = P.last_sig[(size_t)j * n + s];
        float deemph = P.deemph[s];
        int last_exc = P.last_exc[s];
        Kiss99 rng;
        rng.z = P.rng[s]; rng.w = P.rng[(size_t)n + s]; rng.jsr = P.rng[2 * (size_t)n + s]; rng.jcong = P.rng[3 * (size_t)n + s];
        short *pcm_out = P.pcm + (size_t)s * P.pcm_stream_stride;
        int step = 0;
        for (int f = 0; f < P.nframes; f++) {
            {
                const float *lp = P.lpc_raw + ((size_t)f * n + s) * LPC_ORDER;
                const float4 a = ldg4(lp), b = ldg4(lp + 4), c = ldg4(lp + 8), d = ldg4(lp + 12);
                const float raw[16] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
#pragma unroll
                for (int j = 0; j < LPC_ORDER; j++) lpc[j] = __fmul_rn(raw[j], __ldg(&P.gamma_pow[j]));
            }
            for (int t = 0; t < spf; t++, step++) {
                float pred = 0.f;
#pragma unroll
                for (int j = 0; j < LPC_ORDER; j++) pred = __fsub_rn(pred, __fmul_rn(ls[j], lpc[j]));
                idx_s[lane] = lin2ulaw(ls[0]); idx_s[32 + lane] = lin2ulaw(pred); idx_s[64 + lane] = last_exc;
                __threadfence_block();
                bar_arrive(FB_IDX, F_THREADS);
                float thr[8];
                {
                    uint32_t r0 = kiss99_rand(rng), r1 = kiss99_rand(rng);
                    thr[0] = logit[r0 & 0xFF]; thr[1] = logit[(r0 >> 8) & 0xFF]; thr[2] = logit[(r0 >> 16) & 0xFF]; thr[3] = logit[r0 >> 24];
                    thr[4] = logit[r1 & 0xFF]; thr[5] = logit[(r1 >> 8) & 0xFF]; thr[6] = logit[(r1 >> 16) & 0xFF]; thr[7] = logit[r1 >> 24];
                }
                bar_sync(FB_HB, F_THREADS);
                const float *hbn = hBs + ((step & 1) ^ 1) * NB * 32;
                float hbv[NB];
#pragma unroll
                for (int j = 0; j < NB; j++) hbv[j] = hbn[j * 32 + lane];
                int val = 0;
#pragma unroll
                for (int b = 0; b < 8; b++) {
                    const int i = (1 << b) | val;
                    float sum1 = fcb[i], sum2 = fcb[256 + i];
                    const float *wr = P.fcw + i * FCW_ROW;
#pragma unroll
                    for (int j0 = 0; j0 < NB; j0 += 8) {
                        const float4 a0 = ldg4(wr + j0), a1 = ldg4(wr + j0 + 4), c0 = ldg4(wr + NB + j0), c1 = ldg4(wr + NB + j0 + 4);
                        const float wa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w}, wc[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
                        for (int j = 0; j < 8; j++) {
                            sum1 = __fadd_rn(sum1, __fmul_rn(wa[j], hbv[j0 + j]));
                            sum2 = __fadd_rn(sum2, __fmul_rn(wc[j], hbv[j0 + j]));
                        }
                    }
                    sum1 = __fmul_rn(fcf[i], tanh_approx(sum1, rcp));
                    sum2 = __fmul_rn(fcf[256 + i], tanh_approx(sum2, rcp));
                    sum1 = __fadd_rn(sum1, sum2);
                    val = (val << 1) | (thr[b] < sum1 ? 1 : 0);
                }
                int exc = val;
                float pcm;
                const bool forced = f == 0 && t < (P.fast_cvt >> 8);      // `preload` teacher forcing (lpcnet.c:256-259), see SampleParams::fast_cvt
                if (forced) {
                    const float o = (float)pcm_out[t];
                    pcm = __fsub_rn(o, __fmul_rn(0.85f, deemph));
                    exc = lin2ulaw(__fsub_rn(pcm, pred));
                } else pcm = __fadd_rn(pred, u2l[exc]);
#pragma unroll
                for (int j = LPC_ORDER - 1; j > 0; j--) ls[j] = ls[j - 1];
                ls[0] = pcm;
                last_exc = exc;
                pcm = __fadd_rn(pcm, __fmul_rn(0.85f, deemph));
                deemph = pcm;
                if (pcm < -32767) pcm = -32767;
                if (pcm > 32767) pcm = 32767;
                if (live && !forced) pcm_out[(size_t)f * spf + t] = (short)__double2int_rd(0.5 + (double)pcm);
            }
        }
        if (live) {
#pragma unroll
            for (int j = 0; j < LPC_ORDER; j++) P.last_sig[(size_t)j * n + s] = ls[j];
            P.deemph[s] = deemph; P.last_exc[s] = last_exc;
            P.rng[s] = rng.z; P.rng[(size_t)n + s] = rng.w; P.rng[2 * (size_t)n + s] = rng.jsr; P.rng[3 * (size_t)n + s] = rng.jcong;
        }
    }
}

__global__ void __launch_bounds__(F_THREADS, 1) lpcnet_sample_kernel_f32(const __grid_constant__ SampleParams P)
{
    sample_body_f32(P, blockIdx.x);
}

// Several float batches of one GRU_A size in one launch: member k holds CTAs [cta0[k], cta0[k+1]) (GroupSampleParams, engine.h),
// spc live slots each.  Everything that differs between members (image, layout, the dense GRU_B flag, stream count) is read from
// the member's parameters, so members with different sparsity patterns share the launch.
__global__ void __launch_bounds__(F_THREADS, 1) lpcnet_group_sample_kernel_f32(const __grid_constant__ GroupSampleParams G)
{
    const int c = blockIdx.x;
    int k = 0;
#pragma unroll 1
    for (int j = 1; j < G.count; j++) if (c >= G.cta0[j]) k = j;
    sample_body_f32(G.m[k], c - G.cta0[k]);
}

cudaError_t launch_group_sample_kernel_f32(const GroupSampleParams &g, int ctas, uint32_t smem_bytes, cudaStream_t st)
{
    cudaError_t e = cudaFuncSetAttribute(lpcnet_group_sample_kernel_f32, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    lpcnet_group_sample_kernel_f32<<<ctas, F_THREADS, smem_bytes, st>>>(g);
    return cudaGetLastError();
}

cudaError_t launch_sample_kernel_f32(const SampleParams &p, cudaStream_t st)
{
    cudaError_t e = cudaFuncSetAttribute(lpcnet_sample_kernel_f32, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    const int ctas = (p.n_streams + p.spc - 1) / p.spc;
    lpcnet_sample_kernel_f32<<<ctas, F_THREADS, p.L.total_bytes, st>>>(p);
    return cudaGetLastError();
}

}  // namespace LPCNET_KNS
}  // namespace lpcnet_b200
