// frame_kernels.cu — the 100 Hz path: conditioning network, cepstrum->LPC, packet decoder.
//
// Replaces (reference file:line):
//   run_frame_network          src/lpcnet.c:82-120      (embedding, conv1d x2, dense x4 -> gru_a/gru_b condition)
//   compute_conv1d / dense     src/nnet.c:452-470,122-135 over sgemv_accum16 (src/vec_avx.h:618-643)
//   lpc_from_cepstrum          src/freq.c:310-320 (+ idct :230, interp_band_gain :202, inverse_transform :256,
//                              opus_fft_c src/kiss_fft.c:566, lpcn_lpc src/freq.c:86)
//   decode_packet              src/lpcnet_dec.c:81-155, perform_double_interp src/common.c:58-65
//
// Arithmetic contract: every output neuron is ONE thread walking its inputs in ascending order with __fmaf_rn
// (exactly the per-row FMA chain of sgemv_accum16), so results equal the reference build A/B bit for bit.  This
// file is compiled with -fmad=false: plain a*b+c below are separate IEEE operations, as in the pinned oracle build
// (-ffp-contract=off).  ~2.5 % of the MACs of the whole path (SURVEY.md 8a F7): not on the roofline-critical side.
#include <cstdint>
#include "engine.h"
#include "devmath.cuh"
#include "frame_dev.cuh"

namespace lpcnet_b200 {

// The conditioning network is evaluated LAYER BY LAYER over all (stream, frame) columns of a chunk as plain fp32 GEMMs:
// nothing in it is sequential across frames except the 3-frame convolution windows, and those are just overlapping reads of a
// per-stream row buffer that starts with the two carried frames (conv state).  One generic kernel, frame_gemm_kernel:
//   Y[col][i] = act(bias[i] + sum_{j<M} W[j*N+i] * X[col][j]),   j ascending, one fmaf per term, accumulator starts at the bias
// = the per-row FMA chain of sgemv_accum16 (vec_avx.h:618-643) for every output, so the result does not depend on the tiling.
// Block tile 128 outputs x 32 columns x 16 k, 64 threads, thread tile 8 x 8 (64 FFMA per 4 LDS.128: with 8 x 4 tiles the kernel sat
// on the shared-memory pipe); W and X tiles are double-buffered through shared memory (register-staged
// prefetch of the next k-tile while the current one is multiplied).  Small blocks on purpose: a layer has only ~1300 tiles at
// 4096 streams x 10 frames, so many resident blocks per SM keep the SMs evenly loaded.
constexpr int GT_N = 128, GT_C = 32, GT_K = 16, GT_XPAD = 36, GT_THREADS = 64;

struct GemmArgs {
    const float *W, *bias; int M, N, ldw;  // W[j*ldw + i], i < N (reference layout of dense / conv weights: dump_lpcnet.py:194-200,229-245; ldw > N: a column slice)
    const float *X; int xS, xF;            // column (s, f) reads its M inputs at X + ((size_t)s*xS + f)*xF  (conv: overlapping windows, xF < M)
    float *Y; long long ys, yf, y0;        // output i of column (s, f) goes to Y + s*ys + f*yf + y0 + i
    int F, ncols;                          // frames per stream in this call, ncols = n*F
    const int *fc; int zthr;               // output zeroed while frame_count[s] + f < zthr (warm-up, lpcnet.c:99,101); fc == NULL: never
    const uint16_t *rcp16;
};

template <bool TANH>
__global__ void __launch_bounds__(GT_THREADS) frame_gemm_kernel(const GemmArgs a)
{
    __shared__ __align__(16) float Ws[2][GT_K][GT_N];
    __shared__ __align__(16) float Xs[2][GT_K][GT_XPAD];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int c0 = blockIdx.x * GT_C, i0 = blockIdx.y * GT_N;
    // ---- loader roles: X tile = 32 columns x 16 k (thread: columns tid/4 and 16 + tid/4, 4 consecutive k each),
    //      W tile = 16 k x 128 outputs (thread: 8 rows, one float4 each) ----
    const int kq = tid & 3;
    const float *xp[2]; bool xvalid[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int xc = c0 + (tid >> 2) + 16 * h;
        xvalid[h] = xc < a.ncols;
        const int xs_ = xvalid[h] ? xc / a.F : 0, xf_ = xvalid[h] ? xc - (xc / a.F) * a.F : 0;
        xp[h] = a.X + ((size_t)xs_ * a.xS + xf_) * a.xF + 4 * kq;
    }
    const int wq = tid & 31, wr = tid >> 5;
    const bool wvalid = i0 + 4 * wq < a.N;
    const float *wp = a.W + i0 + 4 * wq;
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 wreg[8], xreg[2];
    auto gload = [&](int k0) {
#pragma unroll
        for (int e = 0; e < 8; e++) { const int k = k0 + wr + 2 * e; wreg[e] = (wvalid && k < a.M) ? ldg4(wp + (size_t)k * a.ldw) : zero4; }
#pragma unroll
        for (int h = 0; h < 2; h++) xreg[h] = (xvalid[h] && k0 + 4 * kq < a.M) ? ldg4(xp[h] + k0) : zero4;
    };
    auto sstore = [&](int b) {
#pragma unroll
        for (int e = 0; e < 8; e++) *reinterpret_cast<float4 *>(&Ws[b][wr + 2 * e][4 * wq]) = wreg[e];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int c = (tid >> 2) + 16 * h;
            Xs[b][4 * kq + 0][c] = xreg[h].x; Xs[b][4 * kq + 1][c] = xreg[h].y; Xs[b][4 * kq + 2][c] = xreg[h].z; Xs[b][4 * kq + 3][c] = xreg[h].w;
        }
    };
    // ---- compute roles: warp wn owns 64 outputs x all 32 columns; lane (ln, lc) outputs nA..nA+3, nA+32..nA+35, columns cc..cc+7 ----
    const int wn = warp, ln = lane & 7, lc = lane >> 3;
    const int nA = wn * 64 + ln * 4, cc = lc * 8;
    float acc[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int i = i0 + nA + (r & 3) + (r >> 2) * 32;
        const float b = i < a.N ? __ldg(&a.bias[i]) : 0.f;
#pragma unroll
        for (int c = 0; c < 8; c++) acc[r][c] = b;
    }
    const int nk = (a.M + GT_K - 1) / GT_K;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < nk; kt++) {
        const int b = kt & 1;
        if (kt + 1 < nk) gload((kt + 1) * GT_K);
        const int klen = min(GT_K, a.M - kt * GT_K);          // the last tile of a 252-input layer is short: no zero-padded terms are added
        auto step = [&](int kk) {
            const float4 wa = *reinterpret_cast<const float4 *>(&Ws[b][kk][nA]);
            const float4 wb = *reinterpret_cast<const float4 *>(&Ws[b][kk][nA + 32]);
            const float4 xa = *reinterpret_cast<const float4 *>(&Xs[b][kk][cc]);
            const float4 xb = *reinterpret_cast<const float4 *>(&Xs[b][kk][cc + 4]);
            const float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w}, xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int c = 0; c < 8; c++) acc[r][c] = __fmaf_rn(w[r], xv[c], acc[r][c]);
        };
        if (klen == GT_K) {
#pragma unroll
            for (int kk = 0; kk < GT_K; kk++) step(kk);
        } else {
            for (int kk = 0; kk < klen; kk++) step(kk);
        }
        if (kt + 1 < nk) sstore(b ^ 1);
        __syncthreads();
    }
    // ---- epilogue: activation, warm-up zeroing, store ----
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const int col = c0 + cc + c;
        if (col >= a.ncols) continue;
        const int s = col / a.F, f = col - s * a.F;
        const bool zero = a.fc && __ldg(&a.fc[s]) + f < a.zthr;
        float *yp = a.Y + (size_t)s * a.ys + (size_t)f * a.yf + a.y0 + i0 + nA;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (i0 + nA + 32 * h >= a.N) continue;
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; e++) {
                float y = acc[4 * h + e][c];
                if (TANH) y = tanh_approx_x86(y, a.rcp16);
                v[e] = zero ? 0.f : y;
            }
            *reinterpret_cast<float4 *>(yp + 32 * h) = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

struct FrameIoArgs {
    const float *embed_pitch;
    float *conv1_state, *conv2_state;
    const float *features; long long stream_stride; int frame_stride;
    int n, F;
    int *frame_count;
    float *E1, *E2;          // row buffers [n][F+2][84] / [n][F+2][128]: rows 0,1 = the carried frames (conv state), row 2+f = frame f
    const float *CD;         // [n][F][128] conditioning vectors (END2END: the first 16 are reflection coefficients)
    float *lpc_e2e;          // [F][n][16] or NULL
};

// rc2lpc (lpcnet.c:57-78): reflection coefficients -> direct-form LPC, the reference's exact (unusual) recursion
__device__ __forceinline__ void rc2lpc_dev(float *lpc, const float *rc)
{
    float tmp[LPC_ORDER], ntmp[LPC_ORDER];
    for (int i = 0; i < LPC_ORDER; i++) { tmp[i] = rc[i]; ntmp[i] = 0.f; }
    for (int i = 0; i < LPC_ORDER; i++) {
        for (int j = 0; j <= i - 1; j++) ntmp[j] = __fadd_rn(tmp[j], __fmul_rn(tmp[i], tmp[i - j - 1]));
        for (int k = 0; k <= i - 1; k++) tmp[k] = ntmp[k];
    }
    for (int i = 0; i < LPC_ORDER; i++) lpc[i] = tmp[i];
}

// input assembly (lpcnet.c:93-96): one block per stream fills its rows of E1 (features | pitch embedding) and the carried rows of E1 / E2
__global__ void __launch_bounds__(128) frame_assemble_kernel(const FrameIoArgs a)
{
    const int s = blockIdx.x, tid = threadIdx.x;
    float *e1 = a.E1 + (size_t)s * (a.F + 2) * FRAME_IN, *e2 = a.E2 + (size_t)s * (a.F + 2) * COND;
    for (int e = tid; e < 2 * FRAME_IN; e += blockDim.x) e1[e] = a.conv1_state[(size_t)s * 2 * FRAME_IN + e];
    for (int e = tid; e < 2 * COND; e += blockDim.x) e2[e] = a.conv2_state[(size_t)s * 2 * COND + e];
    for (int e = tid; e < a.F * FRAME_IN; e += blockDim.x) {
        const int f = e / FRAME_IN, j = e - f * FRAME_IN;
        const float *ft = a.features + (size_t)s * a.stream_stride + (size_t)f * a.frame_stride;
        float v;
        if (j < NB_FEAT) v = ft[j];
        else {
            // pitch = (int)floor(.1 + 50*features[NB_BANDS]+100): 50*f is a float product, the sums are double; past int32
            // (f above about 4.3e7, inf) and for NaN x86 gives INT_MIN, which the clamp turns into 33
            int p = cvtt_x86(floor((.1 + (double)__fmul_rn(50.f, ft[NB_BANDS])) + 100.0));
            p = min(255, max(33, p));
            v = __ldg(&a.embed_pitch[p * PITCH_EMBED + (j - NB_FEAT)]);
        }
        e1[(size_t)(2 + f) * FRAME_IN + j] = v;
    }
}

// after the layers: new conv states = the last two rows (mem <- tmp[nb_inputs:], nnet.c:469), frame counters (lpcnet.c:119),
// END2END LPC (lpcnet.c:105,107-108)
__global__ void __launch_bounds__(128) frame_finish_kernel(const FrameIoArgs a)
{
    const int s = blockIdx.x, tid = threadIdx.x;
    const float *e1 = a.E1 + ((size_t)s * (a.F + 2) + a.F) * FRAME_IN, *e2 = a.E2 + ((size_t)s * (a.F + 2) + a.F) * COND;
    for (int e = tid; e < 2 * FRAME_IN; e += blockDim.x) a.conv1_state[(size_t)s * 2 * FRAME_IN + e] = e1[e];
    for (int e = tid; e < 2 * COND; e += blockDim.x) a.conv2_state[(size_t)s * 2 * COND + e] = e2[e];
    if (tid == 0) a.frame_count[s] = min(1000, a.frame_count[s] + a.F);
    if (a.lpc_e2e && tid < a.F) {
        float lp[LPC_ORDER];
        rc2lpc_dev(lp, a.CD + ((size_t)s * a.F + tid) * COND);
        float *o = a.lpc_e2e + ((size_t)tid * a.n + s) * LPC_ORDER;
        for (int i = 0; i < LPC_ORDER; i++) o[i] = lp[i];
    }
}

// ------------------------------------------------------------------------------------------------------------------
// cepstrum -> LPC, one WARP per (frame, stream).  The 320-point complex FFT follows the reference's mixed-radix schedule
// (factors 5,4,4,4: lpcnet_tables.c:200) butterfly for butterfly, so that the 17 autocorrelation lags — and hence the LPCs,
// the prediction and every u-law index derived from it — are bit-identical; the 80 (64) butterflies of a stage are independent
// and are dealt to the lanes, the data lives in shared memory.  IDCT rows and the spectral interpolation are spread over the
// lanes the same way (each output is still one sequential chain); the Levinson recursion is serial and runs on lane 0.
struct LpcArgs {
    const float *features; long long stream_stride; int frame_stride; int n, nframes;
    const float *dct; const c32 *tw; const int16_t *bitrev;
    float *lpc_raw;       // [nframes+2][n][16]; this kernel fills entries 2..nframes+1
};

constexpr int LPC_WARPS = 4;

__global__ void __launch_bounds__(LPC_WARPS * 32) lpc_kernel(const LpcArgs a)
{
    __shared__ c32 ysh[LPC_WARPS][WINDOW_SIZE];
    __shared__ float exsh[LPC_WARPS][NB_BANDS + 2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long gid = (long long)blockIdx.x * LPC_WARPS + warp;
    if (gid >= (long long)a.n * a.nframes) return;               // (whole warps leave; only __syncwarp below)
    const int f = (int)(gid / a.n), s = (int)(gid % a.n);
    const float *cep = a.features + (size_t)s * a.stream_stride + (size_t)f * a.frame_stride;
    float lpc[LPC_ORDER];
    cepstrum_to_lpc_warp(cep, ysh[warp], exsh[warp], a.dct, a.tw, a.bitrev, lpc, lane);
    if (lane != 0) return;
    float *out = a.lpc_raw + ((size_t)(f + 2) * a.n + s) * LPC_ORDER;
#pragma unroll
    for (int i = 0; i < LPC_ORDER; i++) out[i] = lpc[i];
}

// lpc_carry[0] = LPC of frame -1, lpc_carry[1] = frame -2 (old_lpc[0], old_lpc[1] of lpcnet.c:110-112).
// lpc_raw entry e holds the raw LPC of frame e-2, so frame f reads entry f.
__global__ void lpc_carry_in_kernel(const float *carry, float *lpc_raw, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * LPC_ORDER) return;
    lpc_raw[i] = carry[(size_t)n * LPC_ORDER + i];                       // entry 0 = frame -2
    lpc_raw[(size_t)n * LPC_ORDER + i] = carry[i];                       // entry 1 = frame -1
}
__global__ void lpc_carry_out_kernel(float *carry, const float *lpc_raw, int n, int nframes)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * LPC_ORDER) return;
    carry[i] = lpc_raw[(size_t)(nframes + 1) * n * LPC_ORDER + i];              // last frame
    carry[(size_t)n * LPC_ORDER + i] = lpc_raw[(size_t)nframes * n * LPC_ORDER + i];   // the one before
}

// lpc_raw [nframes+2][n][16]: entry e holds the raw (unweighted) LPC of frame e-2 of this call (entries 0,1 = the carry of the
// previous call), so a model with FEATURES_DELAY d reads entry f + 2 - d for frame f (lpcnet.c:109-115); END2END models get the
// network's own LPC of frame f written to entry f + 2 (and are read with d = 0).
void launch_frame_network(const DeviceModel &m, const FrameState &fs, const float *d_features, long long stream_stride,
                          int frame_stride, int n, int nframes, float *condA, float *condB, float *lpc_raw, cudaStream_t st)
{
    const int F = nframes, na3 = 3 * m.na;
    // scratch rows of this chunk (FrameState::work, sized for FRAME_CHUNK frames): E1 [n][F+2][84], E2 [n][F+2][128], P, Q [n][F][128]
    float *E1 = fs.work, *E2 = E1 + (size_t)n * (FRAME_CHUNK + 2) * FRAME_IN, *P = E2 + (size_t)n * (FRAME_CHUNK + 2) * COND, *Q = P + (size_t)n * FRAME_CHUNK * COND;
    FrameIoArgs io{m.embed_pitch, fs.conv1_state, fs.conv2_state, d_features, stream_stride, frame_stride, n, F, fs.frame_count, E1, E2, P,
                   m.cfg.end2end ? lpc_raw + (size_t)2 * n * LPC_ORDER : nullptr};
    // cepstrum -> LPC depends on the features only: it runs on a side stream next to the conditioning network (fork / join by events),
    // so this latency-bound warp-per-frame kernel hides behind the GEMMs instead of adding to the step
    const bool lpc_path = !m.cfg.end2end;                      // END2END: no cepstrum -> LPC path, no delay line (lpcnet.c:107-108)
    const bool fork = lpc_path && fs.side != nullptr;
    cudaStream_t ls = fork ? fs.side : st;
    auto lpc_part = [&]() {
        const int tpb = 128;
        lpc_carry_in_kernel<<<(n * LPC_ORDER + tpb - 1) / tpb, tpb, 0, ls>>>(fs.lpc_carry, lpc_raw, n);
        LpcArgs la{d_features, stream_stride, frame_stride, n, nframes, m.dct, reinterpret_cast<const c32 *>(m.twiddles), m.bitrev, lpc_raw};
        long long tot = (long long)n * nframes;
        lpc_kernel<<<(unsigned)((tot + LPC_WARPS - 1) / LPC_WARPS), LPC_WARPS * 32, 0, ls>>>(la);
        lpc_carry_out_kernel<<<(n * LPC_ORDER + tpb - 1) / tpb, tpb, 0, ls>>>(fs.lpc_carry, lpc_raw, n, nframes);
    };
    if (fork) {
        cudaEventRecord(fs.ev_fork, st);                       // everything queued so far (previous sample kernel reading lpc_raw, H2D of the features) is ordered before
        cudaStreamWaitEvent(fs.side, fs.ev_fork, 0);
        lpc_part();
        cudaEventRecord(fs.ev_join, fs.side);
    }
    frame_assemble_kernel<<<n, 128, 0, st>>>(io);
    const int ncols = n * F;
    auto gemm = [&](bool tanh_act, const float *W, const float *bias, int M, int N, const float *X, int xS, int xF,
                    float *Y, long long ys, long long yf, long long y0, const int *fc, int zthr, int ldw = 0) {
        GemmArgs g{W, bias, M, N, ldw ? ldw : N, X, xS, xF, Y, ys, yf, y0, F, ncols, fc, zthr, m.rcp16};
        dim3 grid((ncols + GT_C - 1) / GT_C, (N + GT_N - 1) / GT_N);
        if (tanh_act) frame_gemm_kernel<true><<<grid, GT_THREADS, 0, st>>>(g);
        else frame_gemm_kernel<false><<<grid, GT_THREADS, 0, st>>>(g);
    };
    // conv1 (nnet.c:452-470; zeroed while frame_count < FEATURE_CONV1_DELAY = 1, lpcnet.c:99): window = rows f..f+2 of E1 -> row 2+f of E2
    gemm(true, m.conv1_w, m.conv1_b, 3 * FRAME_IN, COND, E1, F + 2, FRAME_IN, E2, (long long)(F + 2) * COND, COND, 2 * COND, fs.frame_count, 1);
    // conv2 (zeroed while frame_count < FEATURES_DELAY, lpcnet.c:101)
    gemm(true, m.conv2_w, m.conv2_b, 3 * COND, COND, E2, F + 2, COND, P, (long long)F * COND, COND, 0, fs.frame_count, m.cfg.features_delay);
    gemm(true, m.dense1_w, m.dense1_b, COND, COND, P, F, COND, Q, (long long)F * COND, COND, 0, nullptr, 0);
    gemm(true, m.dense2_w, m.dense2_b, COND, COND, Q, F, COND, P, (long long)F * COND, COND, 0, nullptr, 0);
    // gru_a_dense_feature (128 -> 3*na, linear) and gru_b_dense_feature (128 -> 48, linear): outputs frame-major [f][n][.]
    if (m.is_float) gemm(false, m.gad_w, m.gad_b, COND, na3, P, F, COND, condA, na3, (long long)n * na3, 0, nullptr, 0);
    else {
        // int8 flavour: one GEMM per gate (a column slice of the weight matrix) into the gate-major, tile-pitched layout (condA_frame_floats)
        const long long crow = m.na + 8, fA = (long long)condA_frame_floats(false, (size_t)n, m.na);
        for (int g = 0; g < 3; g++)
            gemm(false, m.gad_w + (size_t)g * m.na, m.gad_b + (size_t)g * m.na, COND, m.na, P, F, COND, condA + (size_t)g * n * crow, crow, fA, 0, nullptr, 0, na3);
    }
    gemm(false, m.gbd_w, m.gbd_b, COND, 3 * NB, P, F, COND, condB, 3 * NB, (long long)n * 3 * NB, 0, nullptr, 0);
    frame_finish_kernel<<<n, 128, 0, st>>>(io);
    if (fork) cudaStreamWaitEvent(st, fs.ev_join, 0);
    else if (lpc_path) lpc_part();
}
int frame_network_launches(const DeviceModel &m) { return (m.cfg.end2end ? 8 : 11) + (m.is_float ? 0 : 2); }
size_t frame_work_floats(size_t n) { return n * ((size_t)(FRAME_CHUNK + 2) * (FRAME_IN + COND) + 2 * (size_t)FRAME_CHUNK * COND); }

// ------------------------------------------------------------------------------------------------------------------
// decode_packet (lpcnet_dec.c:81-155): 64-bit packet -> 4 feature frames; one thread per stream, packets in order
// (vq_mem carries across packets).
struct DecodeArgs { const uint8_t *packets; int n, npackets; const float *cb; const float *pitch_pow; float *vq_mem; float *features; };

__global__ void decode_kernel(const DecodeArgs a)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const float *cb1 = a.cb, *cb2 = cb1 + 1024 * 17, *cb3 = cb2 + 1024 * 17, *cbd4 = cb3 + 1024 * 17;
    float vq_mem[NB_BANDS];
    for (int i = 0; i < NB_BANDS; i++) vq_mem[i] = a.vq_mem[(size_t)s * NB_BANDS + i];
    for (int p = 0; p < a.npackets; p++) {
        const uint8_t *buf = a.packets + ((size_t)s * a.npackets + p) * 8;
        unsigned long long bits = 0;
        for (int i = 0; i < 8; i++) bits = (bits << 8) | buf[i];                  // MSB-first, bits_unpack :59-78
        int pos = 0;
        auto get = [&](int nb) { pos += nb; return (int)((bits >> (64 - pos)) & ((1ull << nb) - 1)); };
        int c0_id = get(7), main_pitch = get(6), modulation = get(3), corr_id = get(2);
        int vq0 = get(10), vq1 = get(10), vq2 = get(10), vq_mid = get(13), interp_id = get(3);
        float *F = a.features + ((size_t)s * a.npackets + p) * 4 * NB_FEAT;      // [4][20]
        float f1[NB_BANDS], f3[NB_BANDS];
        int voiced = 1;
        modulation -= 4;
        if (modulation == -4) { voiced = 0; modulation = 0; }
        float frame_corr = voiced ? 0.3875f + .175f * corr_id : 0.0375f + .075f * corr_id;
        for (int sub = 0; sub < 4; sub++) {
            float pch = a.pitch_pow[main_pitch];                                  // (float)(pow(2.f, main_pitch/21.)*PITCH_MIN_PERIOD)
            pch *= 1.f + __fdiv_rn(__fdiv_rn((float)modulation, 16.f), 7.f) * (2 * sub - 3);
            float mx = 33 > pch ? 33.f : pch;                                     // MIN16(255, MAX16(33, p))
            pch = 255 < mx ? 255.f : mx;
            F[sub * NB_FEAT + NB_BANDS] = .02f * (pch - 100.f);
            F[sub * NB_FEAT + NB_BANDS + 1] = frame_corr - .5f;
        }
        f3[0] = __fdiv_rn((float)(c0_id - 64), 4.f);
        for (int i = 0; i < NB_BANDS - 1; i++) f3[i + 1] = cb1[vq0 * 17 + i] + cb2[vq1 * 17 + i] + cb3[vq2 * 17 + i];
        float sign = 1;
        if (vq_mid >= 4096) { vq_mid -= 4096; sign = -1; }
        for (int i = 0; i < NB_BANDS; i++) f1[i] = sign * cbd4[vq_mid * NB_BANDS + i];
        if ((vq_mid & 3) < 2) { for (int i = 0; i < NB_BANDS; i++) f1[i] += .5f * (vq_mem[i] + f3[i]); }
        else if ((vq_mid & 3) == 2) { for (int i = 0; i < NB_BANDS; i++) f1[i] += vq_mem[i]; }
        else { for (int i = 0; i < NB_BANDS; i++) f1[i] += f3[i]; }
        interp_id += (interp_id >= 7);                                            // FORBIDDEN_INTERP, common.c:58-65
        const int id0 = interp_id / 3, id1 = interp_id % 3;
        for (int i = 0; i < NB_BANDS; i++) {
            F[0 * NB_FEAT + i] = id0 == 0 ? .5f * (vq_mem[i] + f1[i]) : (id0 == 1 ? vq_mem[i] : f1[i]);
            F[1 * NB_FEAT + i] = f1[i];
            F[2 * NB_FEAT + i] = id1 == 0 ? .5f * (f1[i] + f3[i]) : (id1 == 1 ? f1[i] : f3[i]);
            F[3 * NB_FEAT + i] = f3[i];
            vq_mem[i] = f3[i];
        }
    }
    for (int i = 0; i < NB_BANDS; i++) a.vq_mem[(size_t)s * NB_BANDS + i] = vq_mem[i];
}

void launch_decode_packets(const DeviceModel &m, const FrameState &fs, const uint8_t *d_packets, int n, int npackets,
                           float *d_features, cudaStream_t st)
{
    DecodeArgs da{d_packets, n, npackets, m.codebooks, m.pitch_pow, fs.vq_mem, d_features};
    decode_kernel<<<(n + 127) / 128, 128, 0, st>>>(da);
}

}  // namespace lpcnet_b200
