// sample_kernel_f32n.cu — float flavour of the per-sample loop for SMALL batches: one GRU_A neuron per lane.
//
// Same arithmetic, operation for operation, as sample_kernel_f32.cu (reference float build B: per-row sequential fp32 FMA
// chains in block order, src/vec_avx.h:760-788 / src/nnet.c:326-372,410-448), different mapping: with a handful of streams
// per SM (BASELINE config 2: 256 streams on 148 SMs) lane==stream leaves 30 of 32 lanes idle while each busy lane walks
// every chain of its warp's 24 neurons.  Here
//   * compute lane (warp w, lane l) owns neuron FNI_NEUR[32w + l] of GRU_A: its r, h and z rows are three sequential FMA
//     chains over the row group's block lists; the 8 lanes of a row group read the same state vector (LDS.128 broadcast)
//     and their own 8 bytes of each fp16 block (LDS.64).  Up to FN_S streams per CTA give the independent chains that
//     hide the FMA latency.  Gate activations and the state update need no exchange: the lane holds all three rows.
//   * the conditioning inputs are read directly, coalesced across the 384 neuron lanes (no gather tiles),
//   * the 48 rows of GRU_B (384-term chains, the longest serial piece of a sample) run on 48 lanes, then 16 x S lanes finish,
//   * one sampler warp, lane == stream (same code as the other float kernel).
#include <cstdint>
#include <cuda_fp16.h>
#ifndef LPCNET_NA
#define LPCNET_NA 384          // GRU_A units this translation unit is compiled for
#endif
#include "sample_common.cuh"

namespace lpcnet_b200 {
namespace LPCNET_KNS {

namespace {

enum { NB_IDX = 1, NB_X = 2, NB_ACCB = 3, NB_HB = 4 };
constexpr int CNT_ALL = FN_THREADS, CNT_CMP = FN_NWC * 32;

// y[s] = fma(w[c], x[s][pos + c], y[s]), c = 0..3, for the blocks of this lane's row, in list order (one row of
// sparse_sgemv_accum8x4 / sgemv_accum8x4, float).  `nb` is this lane's list length, `nbmax` the longest list in the warp
// (the loop bound must be warp-uniform); w = this lane's 8 bytes of the first block, meta = the list's first meta entry.
// Blocks go in pairs through a software pipeline: while pair p is multiplied, the operands of pair p+1 and the meta entries
// of pair p+2 are in flight (lanes past the end of their list re-read its last block; those values are never used).
template <int S> struct BlkOps { uint2 w; float4 xv[S]; };
// the four FMAs of one block; `take` = the block belongs to this lane's list (a select, not a branch: a branch per block
// would fence the loads of the software pipeline)
template <int S>
__device__ __forceinline__ void fma_block(float (&y)[FN_S], const BlkOps<S> &o, bool take)
{
    const float2 w01 = __half22float2(*reinterpret_cast<const __half2 *>(&o.w.x)), w23 = __half22float2(*reinterpret_cast<const __half2 *>(&o.w.y));
#pragma unroll
    for (int s = 0; s < S; s++) {
        float v = __fmaf_rn(w01.x, o.xv[s].x, y[s]);
        v = __fmaf_rn(w01.y, o.xv[s].y, v);
        v = __fmaf_rn(w23.x, o.xv[s].z, v);
        v = __fmaf_rn(w23.y, o.xv[s].w, v);
        y[s] = take ? v : y[s];
    }
}
// UNIFORM: every lane of the warp has the same list length (GRU_B rows), no clamping, no select; DENSE: the list is all
// column blocks in order, the state offset of block b is 16*b (no meta look-up in front of the state load)
template <int S, bool UNIFORM, bool DENSE = false>
__device__ __forceinline__ void chain(float (&y)[FN_S], const uint8_t *__restrict__ w, const uint16_t *__restrict__ meta, int nb, int nbmax,
                                      const uint8_t *__restrict__ x /* state buffer, stream 0 */)
{
    const int last = max(nb - 1, 0);
    auto ldm = [&](int b) { return DENSE ? (uint32_t)(16 * min(b, NA / 4 - 1)) : (uint32_t)meta[UNIFORM ? b : min(b, last)]; };
    auto ldb = [&](int b, uint32_t m, BlkOps<S> &o) {
        o.w = *reinterpret_cast<const uint2 *>(w + (size_t)(UNIFORM ? b : min(b, last)) * 64);
#pragma unroll
        for (int s = 0; s < S; s++) o.xv[s] = *reinterpret_cast<const float4 *>(x + m + s * NA * 4);
    };
    uint32_t m2 = ldm(2), m3 = ldm(3);
    BlkOps<S> A0, A1;
    ldb(0, ldm(0), A0); ldb(1, ldm(1), A1);
#pragma unroll 2
    for (int b = 0; b < nbmax; b += 2) {
        BlkOps<S> B0, B1;
        ldb(b + 2, m2, B0); ldb(b + 3, m3, B1);
        m2 = ldm(b + 4); m3 = ldm(b + 5);
        fma_block<S>(y, A0, b < nb);
        fma_block<S>(y, A1, b + 1 < nb);
        A0 = B0; A1 = B1;
    }
}

// the streams of `P` that CTA `cta` of their batch holds: blockIdx.x in a single-batch launch, the member-local CTA index in a
// group launch
template <int S>
__device__ __forceinline__ void run(const SampleParams &P, uint8_t *smem, int cta)
{
    const SmemLayout &L = P.L;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = P.n_streams;
    const int cta_s0 = cta * S;
    const int spf = P.spf;

    const uint32_t bar = smem_u32(smem + FN_MBAR);
    if (threadIdx.x == 0) { mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    if (threadIdx.x == 0) stage_image(smem_u32(smem + FN_IMAGE), P.image, L.image_bytes, bar);
    const uint16_t *rcp = reinterpret_cast<const uint16_t *>(smem + FN_IMAGE + FNI_RCP);
    float *xs = reinterpret_cast<float *>(smem + FN_X);            // [2][FN_S][NA]
    float *hBs = reinterpret_cast<float *>(smem + FN_HB);          // [2][NB][FN_S]
    float *accB = reinterpret_cast<float *>(smem + FN_ACCB);       // [48][FN_S]
    int *idx_s = reinterpret_cast<int *>(smem + FN_IDX);           // [3][FN_S]
    mbar_wait(bar, 0);

    // global stream of slot s (dead slots shadow the batch's last stream: loads valid, stores masked)
    int gs[S]; bool lv[S];
#pragma unroll
    for (int s = 0; s < S; s++) { const int g = cta_s0 + s; lv[s] = g < n; gs[s] = min(g, n - 1); }

    if (warp < FN_NWC) {
        // ================================================= compute warps: lane = neuron j =================================================
        const int cl = warp * 32 + lane;
        const int j = reinterpret_cast<const uint16_t *>(smem + FN_IMAGE + FNI_NEUR)[cl], g = j >> 3, row = j & 7;
        const uint32_t *dirA = reinterpret_cast<const uint32_t *>(smem + FN_IMAGE + FNI_DIRA) + g * 6;
        const float *parA = reinterpret_cast<const float *>(smem + FN_IMAGE + FNI_PARA);
        const uint8_t *wA = smem + L.wA + row * 8;
        const uint16_t *metaA = reinterpret_cast<const uint16_t *>(smem + L.metaA);
        const float bz = parA[0 * NA + j], dz = parA[1 * NA + j], br = parA[2 * NA + j], dr = parA[3 * NA + j], bh = parA[4 * NA + j], dh = parA[5 * NA + j];
        const int fz = (int)dirA[0], nz = (int)dirA[1], fr = (int)dirA[2], nr = (int)dirA[3], fh = (int)dirA[4], nh = (int)dirA[5];
        const int mz = __reduce_max_sync(0xffffffffu, nz), mr = __reduce_max_sync(0xffffffffu, nr), mh = __reduce_max_sync(0xffffffffu, nh);
        // GRU_B input rows: lanes 0..47 of the compute warps 0,1
        const int rowB = cl % (3 * NB);                               // (lanes 48..63 of warp 1 repeat rows 0..15: same list length for the whole warp; not stored)
        const uint32_t *dirB = reinterpret_cast<const uint32_t *>(smem + FN_IMAGE + FNI_DIRB) + (rowB >> 3) * 2;
        const uint8_t *wB = smem + L.wB + (rowB & 7) * 8;
        const uint16_t *metaB = reinterpret_cast<const uint16_t *>(smem + L.metaB);
        const float *parB = reinterpret_cast<const float *>(smem + FN_IMAGE + FNI_PARB);
        const float *wBrec = reinterpret_cast<const float *>(smem + FN_IMAGE + FNI_WBREC);
        // GRU_B finishing lanes: (neuron jb, stream sb): lanes 0 .. 16*S - 1 of the compute warps
        const int jb = cl & 15, sb = min(cl >> 4, S - 1);
        const bool fin = cl < NB * S;

        float h[S];
#pragma unroll
        for (int s = 0; s < S; s++) { h[s] = P.hA[(size_t)j * n + gs[s]]; xs[s * NA + j] = h[s]; }
        float hb = P.hB[(size_t)jb * n + gs[sb]];
        if (fin) hBs[jb * FN_S + sb] = hb;
        bar_sync(NB_X, CNT_CMP);

        int step = 0;
        for (int f = 0; f < P.nframes; f++) {
            float cz[S], cr[S], ch[S];                                  // conditioning of the frame (constant over its samples)
#pragma unroll
            for (int s = 0; s < S; s++) {
                const float *c = P.condA + ((size_t)f * n + gs[s]) * (3 * NA) + j;
                cz[s] = __ldg(c); cr[s] = __ldg(c + NA); ch[s] = __ldg(c + 2 * NA);
            }
            for (int t = 0; t < spf; t++, step++) {
                const int cur = step & 1, nxt = cur ^ 1;
                const uint8_t *xc = reinterpret_cast<const uint8_t *>(xs + cur * FN_S * NA);
                bar_sync(NB_IDX, CNT_ALL);                              // indices of this sample are in idx_s
                float gz[S], gr[S], gh[S];
#pragma unroll
                for (int s = 0; s < S; s++) {                           // compute_gru_a_input (nnet.c:484-491), left to right
                    const float *e0 = P.emb_sig + (size_t)idx_s[s] * (3 * NA) + j;
                    const float *e1 = P.emb_pred + (size_t)idx_s[FN_S + s] * (3 * NA) + j;
                    const float *e2 = P.emb_exc + (size_t)idx_s[2 * FN_S + s] * (3 * NA) + j;
                    gz[s] = __fadd_rn(__fadd_rn(__fadd_rn(cz[s], __ldg(e0)), __ldg(e1)), __ldg(e2));
                    gr[s] = __fadd_rn(__fadd_rn(__fadd_rn(cr[s], __ldg(e0 + NA)), __ldg(e1 + NA)), __ldg(e2 + NA));
                    gh[s] = __fadd_rn(__fadd_rn(__fadd_rn(ch[s], __ldg(e0 + 2 * NA)), __ldg(e1 + 2 * NA)), __ldg(e2 + 2 * NA));
                }
                float y[FN_S], yh[FN_S], r[S], hc[S];
                // candidate pre-activation first (nnet.c:436-440): its chain starts from bias + diag*h and does not need the
                // gathered inputs, so it runs while those loads are in flight
#pragma unroll
                for (int s = 0; s < S; s++) yh[s] = __fadd_rn(bh, __fmul_rn(dh, h[s]));
                chain<S, false>(yh, wA + (size_t)fh * 64, metaA + fh, nh, mh, xc);
                // reset gate (nnet.c:431-435): chain starts from bias + diag*h + gin
#pragma unroll
                for (int s = 0; s < S; s++) y[s] = __fadd_rn(__fadd_rn(br, __fmul_rn(dr, h[s])), gr[s]);
                chain<S, false>(y, wA + (size_t)fr * 64, metaA + fr, nr, mr, xc);
#pragma unroll
                for (int s = 0; s < S; s++) r[s] = sigmoid_approx(y[s], rcp);
                // candidate (nnet.c:441-445)
#pragma unroll
                for (int s = 0; s < S; s++) hc[s] = tanh_approx(__fadd_rn(__fmul_rn(yh[s], r[s]), gh[s]), rcp);
                // update gate and new state (nnet.c:446-447)
#pragma unroll
                for (int s = 0; s < S; s++) y[s] = __fadd_rn(__fadd_rn(bz, __fmul_rn(dz, h[s])), gz[s]);
                chain<S, false>(y, wA + (size_t)fz * 64, metaA + fz, nz, mz, xc);
#pragma unroll
                for (int s = 0; s < S; s++) {
                    const float z = sigmoid_approx(y[s], rcp);
                    h[s] = __fadd_rn(__fmul_rn(z, h[s]), __fmul_rn(__fsub_rn(1.f, z), hc[s]));
                    xs[(nxt * FN_S + s) * NA + j] = h[s];               // other buffer: the chains of other lanes still read the old state
                }
                bar_sync(NB_X, CNT_CMP);
                // GRU_B input side (nnet.c:346-352): one 384-term chain per row, lanes 0..47
                if (warp < 2) {
                    const int nbB = (int)dirB[1], mB = __reduce_max_sync(0xffffffffu, nbB), uB = __reduce_min_sync(0xffffffffu, nbB) == mB;
                    const float *condBp = P.condB + (size_t)f * n * (3 * NB) + rowB;
#pragma unroll
                    for (int s = 0; s < S; s++) y[s] = __fadd_rn(parB[rowB], __ldg(condBp + (size_t)gs[s] * (3 * NB)));
                    const uint8_t *xn = reinterpret_cast<const uint8_t *>(xs + nxt * FN_S * NA);
                    if (uB && L.wBrecF) chain<S, true, true>(y, wB + (size_t)dirB[0] * 64, metaB + dirB[0], nbB, mB, xn);
                    else if (uB) chain<S, true>(y, wB + (size_t)dirB[0] * 64, metaB + dirB[0], nbB, mB, xn);     // all lists alike
                    else chain<S, false>(y, wB + (size_t)dirB[0] * 64, metaB + dirB[0], nbB, mB, xn);
                    if (cl < 3 * NB) {
#pragma unroll
                        for (int s = 0; s < S; s++) accB[rowB * FN_S + s] = y[s];
                    }
                }
                bar_sync(NB_ACCB, CNT_CMP);
                if (fin) {   // GRU_B finish for (neuron jb, stream sb): recurrent chains (sgemv_accum16), gates (nnet.c:353-371)
                    const float *hbo = hBs + cur * NB * FN_S;
                    float rz = parB[3 * NB + jb], rr = parB[4 * NB + jb], rh = parB[5 * NB + jb];
#pragma unroll
                    for (int k = 0; k < NB; k++) {
                        const float xk = hbo[k * FN_S + sb];
                        rz = __fmaf_rn(wBrec[k * 3 * NB + jb], xk, rz);
                        rr = __fmaf_rn(wBrec[k * 3 * NB + NB + jb], xk, rr);
                        rh = __fmaf_rn(wBrec[k * 3 * NB + 2 * NB + jb], xk, rh);
                    }
                    const float zz = sigmoid_approx(__fadd_rn(accB[jb * FN_S + sb], rz), rcp);
                    const float rrr = sigmoid_approx(__fadd_rn(accB[(NB + jb) * FN_S + sb], rr), rcp);
                    const float hh = tanh_approx(__fadd_rn(accB[(2 * NB + jb) * FN_S + sb], __fmul_rn(rh, rrr)), rcp);
                    hb = __fadd_rn(__fmul_rn(zz, hb), __fmul_rn(__fsub_rn(1.f, zz), hh));
                    hBs[nxt * NB * FN_S + jb * FN_S + sb] = hb;
                }
                __threadfence_block();
                bar_arrive(NB_HB, CNT_ALL);
            }
        }
#pragma unroll
        for (int s = 0; s < S; s++) if (lv[s]) P.hA[(size_t)j * n + gs[s]] = h[s];
        if (fin && lv[sb]) P.hB[(size_t)jb * n + gs[sb]] = hb;
    } else {
        // ================================================= sampler warp: lane == stream (same arithmetic as the int8 kernel) =================================================
        const int sl = min(lane, S - 1);
        const bool live = lane < S && lv[sl];
        const int s = gs[sl];
        const float *logit = reinterpret_cast<const float *>(smem + FN_IMAGE + FNI_LOGIT);
        const float *u2l = reinterpret_cast<const float *>(smem + FN_IMAGE + FNI_U2L);
        const float *fcw = reinterpret_cast<const float *>(smem + FN_IMAGE + FNI_FCW);
        float ls[LPC_ORDER], lpc[LPC_ORDER];
#pragma unroll
        for (int k = 0; k < LPC_ORDER; k++) ls[k] = P.last_sig[(size_t)k * n + s];
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
                for (int k = 0; k < LPC_ORDER; k++) lpc[k] = __fmul_rn(raw[k], __ldg(&P.gamma_pow[k]));
            }
            for (int t = 0; t < spf; t++, step++) {
                float pred = 0.f;
#pragma unroll
                for (int k = 0; k < LPC_ORDER; k++) pred = __fsub_rn(pred, __fmul_rn(ls[k], lpc[k]));
                if (lane < S) { idx_s[lane] = lin2ulaw(ls[0]); idx_s[FN_S + lane] = lin2ulaw(pred); idx_s[2 * FN_S + lane] = last_exc; }
                __threadfence_block();
                bar_arrive(NB_IDX, CNT_ALL);
                float thr[8];
                {
                    uint32_t r0 = kiss99_rand(rng), r1 = kiss99_rand(rng);
                    thr[0] = logit[r0 & 0xFF]; thr[1] = logit[(r0 >> 8) & 0xFF]; thr[2] = logit[(r0 >> 16) & 0xFF]; thr[3] = logit[r0 >> 24];
                    thr[4] = logit[r1 & 0xFF]; thr[5] = logit[(r1 >> 8) & 0xFF]; thr[6] = logit[(r1 >> 16) & 0xFF]; thr[7] = logit[r1 >> 24];
                }
                bar_sync(NB_HB, CNT_ALL);
                const float *hbn = hBs + ((step & 1) ^ 1) * NB * FN_S;
                float hbv[NB];
#pragma unroll
                for (int k = 0; k < NB; k++) hbv[k] = hbn[k * FN_S + sl];
                int val = 0;
#pragma unroll
                for (int b = 0; b < 8; b++) {                            // sample_mdense, nnet.c:186-211
                    const int i = (1 << b) | val;
                    const float *wr = fcw + i * FCW_ROW;                  // all 256 rows live in shared memory here
                    const float4 bf = *reinterpret_cast<const float4 *>(wr + 2 * NB);
                    float sum1 = bf.x, sum2 = bf.y;
#pragma unroll
                    for (int j0 = 0; j0 < NB; j0 += 8) {
                        const float4 a0 = *reinterpret_cast<const float4 *>(wr + j0), a1 = *reinterpret_cast<const float4 *>(wr + j0 + 4);
                        const float4 c0 = *reinterpret_cast<const float4 *>(wr + NB + j0), c1 = *reinterpret_cast<const float4 *>(wr + NB + j0 + 4);
                        const float wa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w}, wc[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
                        for (int k = 0; k < 8; k++) {
                            sum1 = __fadd_rn(sum1, __fmul_rn(wa[k], hbv[j0 + k]));
                            sum2 = __fadd_rn(sum2, __fmul_rn(wc[k], hbv[j0 + k]));
                        }
                    }
                    sum1 = __fmul_rn(bf.z, tanh_approx(sum1, rcp));
                    sum2 = __fmul_rn(bf.w, tanh_approx(sum2, rcp));
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
                for (int k = LPC_ORDER - 1; k > 0; k--) ls[k] = ls[k - 1];
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
            for (int k = 0; k < LPC_ORDER; k++) P.last_sig[(size_t)k * n + s] = ls[k];
            P.deemph[s] = deemph; P.last_exc[s] = last_exc;
            P.rng[s] = rng.z; P.rng[(size_t)n + s] = rng.w; P.rng[2 * (size_t)n + s] = rng.jsr; P.rng[3 * (size_t)n + s] = rng.jcong;
        }
    }
}

}  // namespace

template <int S>
__global__ void __launch_bounds__(FN_THREADS, 1) lpcnet_sample_kernel_f32n(const __grid_constant__ SampleParams P)
{
    extern __shared__ __align__(128) uint8_t smem[];
    run<S>(P, smem, blockIdx.x);
}

// Several float batches of one GRU_A size in one launch: member k holds CTAs [cta0[k], cta0[k+1]) (GroupSampleParams, engine.h),
// S streams each.  Every m[k] carries the member's neuron-per-lane layout and image (DeviceModel::Ln / image_n).
template <int S>
__global__ void __launch_bounds__(FN_THREADS, 1) lpcnet_group_sample_kernel_f32n(const __grid_constant__ GroupSampleParams G)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const int c = blockIdx.x;
    int k = 0;
#pragma unroll 1
    for (int j = 1; j < G.count; j++) if (c >= G.cta0[j]) k = j;
    run<S>(G.m[k], smem, c - G.cta0[k]);
}

cudaError_t launch_sample_kernel_f32n(const SampleParams &p, cudaStream_t st)
{
    void (*kern)(SampleParams) = p.spc <= 1 ? lpcnet_sample_kernel_f32n<1> : p.spc == 2 ? lpcnet_sample_kernel_f32n<2> : lpcnet_sample_kernel_f32n<FN_S>;
    const int S = p.spc <= 1 ? 1 : p.spc == 2 ? 2 : FN_S;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    const int ctas = (p.n_streams + S - 1) / S;
    kern<<<ctas, FN_THREADS, p.L.total_bytes, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_group_sample_kernel_f32n(const GroupSampleParams &g, int ctas, uint32_t smem_bytes, cudaStream_t st)
{
    const int spc = g.m[0].spc;                                   // (the same in every member: the group's plan)
    void (*kern)(GroupSampleParams) = spc <= 1 ? lpcnet_group_sample_kernel_f32n<1> : spc == 2 ? lpcnet_group_sample_kernel_f32n<2>
                                                                                               : lpcnet_group_sample_kernel_f32n<FN_S>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    kern<<<ctas, FN_THREADS, smem_bytes, st>>>(g);
    return cudaGetLastError();
}

}  // namespace LPCNET_KNS
}  // namespace lpcnet_b200
