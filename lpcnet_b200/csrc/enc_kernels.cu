// enc_kernels.cu — the analysis side (SURVEY 8f N2): feature extraction and the 1.6 kb/s encoder, batched over streams.
//
// Replaces (reference file:line):
//   lpcnet_compute_single_frame_features(_float)  src/lpcnet_enc.c:911-933  (what `lpcnet_demo -features` runs)
//   lpcnet_encode                                 src/lpcnet_enc.c:882-894  (`lpcnet_demo -encode`)
//   lpcnet_compute_features                       src/lpcnet_enc.c:896-909
//     preemphasis :872, compute_frame_features :498-577 (frame_analysis :488, apply_window freq.c:322, forward_transform freq.c:242,
//     lpcn_compute_band_energy freq.c:131-154, dct freq.c:218, lpc_from_cepstrum freq.c:310, celt_pitch_xcorr pitch.c:44,
//     celt_inner_prod pitch.h:109), process_single_frame :814-870, process_superframe :579-744, quantize_3stage_mbest :133-241,
//     vq_quantize_mbest :53-78, quantize_diff :283-318, find_nearest_multi :243-280, double_interp_search :379-401,
//     perform_double_interp common.c:58-65, bits_pack :443-463.
//
// One block of 256 threads per stream; the stream's LPCNetEncState (lpcnet_private.h:55-75) lives in shared memory for the call.
// Frames of a stream are sequential (analysis overlap, pitch history, Viterbi state); streams are independent.  Every value is
// produced by the reference's own expression in the reference's order (sums are sequential chains in fp32, products and sums
// are separate operations: the library is compiled with -fmad=false like the pinned reference build's -ffp-contract=off), so the
// features and the packets equal the reference's bit for bit; the independent pieces (window, FFT butterflies, bands, the
// 256 lags of the pitch correlation, Viterbi states, codebook distances) are dealt to the threads.
// The three libm calls in double (log10 :516, log :676, pow freq.c:318) use CUDA's double routines.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "engine.h"
#include "frame_dev.cuh"
#include "../../include/lpcnet_b200.h"

namespace lpcnet_b200 {

constexpr int ENC_THREADS = 256;
constexpr int PMAX = 256, PMIN = 32;                 // PITCH_MAX_PERIOD, PITCH_MIN_PERIOD (lpcnet_private.h:14-15)
constexpr int NTOT = 36;                             // NB_TOTAL_FEATURES
constexpr int XC_ROW = PMAX + 1;
constexpr int TRAINING_OFFSET_SAMPLES = 80;          // TRAINING_OFFSET (freq.h:44)

struct EncState {                                    // the fields of struct LPCNetEncState that the three entry points touch
    float analysis_mem[FRAME_SIZE];
    float mem_preemph;
    int pcount;
    float pitch_mem[LPC_ORDER];
    float pitch_filt;
    float xc[10][XC_ROW];
    float frame_weight[10];
    float exc_buf[PMAX + 2 * FRAME_SIZE];
    float pmp[2][PMAX];                              // pitch_max_path
    float pmp_all;
    int best_i;
    float vq_mem[NB_BANDS];
    float features[4][NTOT];
};
constexpr int ENC_STATE_WORDS = sizeof(EncState) / 4;

struct EncTables {
    const float *half_window;     // [160]
    const float *dct;             // [18*18]
    const c32 *tw; const int16_t *bitrev;
    const float *pitch_pow;       // [64] (float)(pow(2.f, k/21.)*32)
    const float *cb;              // ceps_codebook1..3 [1024][17], ceps_codebook_diff4 [4096][18] or NULL
};

struct EncArgs {
    EncState *state; int n;
    const short *pcm16; const float *pcmf;   // exactly one non-NULL: [n][units * samples per unit]
    int units;                               // frames (mode 0) or packets of 4 frames (modes 1, 2)
    float *features;                         // mode 0: [n][units][36]; mode 2: [n][units*4][36]
    unsigned char *packets;                  // mode 1: [n][units][8]
    EncTables t;
};

struct EncScratch {
    c32 y[WINDOW_SIZE];
    float in[FRAME_SIZE], aligned[FRAME_SIZE], sums[FRAME_SIZE + 1];
    float xcorr[PMAX], tmp[PMAX], en[PMAX];
    float Ex[NB_BANDS + 2], Ly[NB_BANDS], lpc[LPC_ORDER];
    unsigned char pitch_prev[8][PMAX];
    float red_d[ENC_THREADS / 32]; int red_i[ENC_THREADS / 32];
    float vq_x[NB_BANDS], vq_target[4 * NB_BANDS], vq_pred[4 * NB_BANDS];
    float sel_d; int sel_i;
    int best[10];
    float frame_corr;
};

#define MAXF(a, b) ((a) > (b) ? (a) : (b))          /* MAX16 / MIN16 of arch.h:72-73 (the comparison decides, also for ties) */
#define MINF(a, b) ((a) < (b) ? (a) : (b))

// block-wide lexicographic minimum of (d, i): the strict `<` scans of the reference keep the first (lowest index) of equal distances
__device__ __forceinline__ void block_argmin(float d, int i, EncScratch &S, float &d_out, int &i_out)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float d2 = __shfl_xor_sync(0xffffffffu, d, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
        if (d2 < d || (d2 == d && i2 < i)) { d = d2; i = i2; }
    }
    if (lane == 0) { S.red_d[warp] = d; S.red_i[warp] = i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float bd = S.red_d[0]; int bi = S.red_i[0];
        for (int w = 1; w < ENC_THREADS / 32; w++) if (S.red_d[w] < bd || (S.red_d[w] == bd && S.red_i[w] < bi)) { bd = S.red_d[w]; bi = S.red_i[w]; }
        S.sel_d = bd; S.sel_i = bi;
    }
    __syncthreads();
    d_out = S.sel_d; i_out = S.sel_i;
    __syncthreads();
}
// the same with the LARGEST value and the lowest index among equals (`if (v > max)` scans)
__device__ __forceinline__ void block_argmax(float v, int i, EncScratch &S, float &v_out, int &i_out)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
        if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
    }
    if (lane == 0) { S.red_d[warp] = v; S.red_i[warp] = i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float bv = S.red_d[0]; int bi = S.red_i[0];
        for (int w = 1; w < ENC_THREADS / 32; w++) if (S.red_d[w] > bv || (S.red_d[w] == bv && S.red_i[w] < bi)) { bv = S.red_d[w]; bi = S.red_i[w]; }
        S.sel_d = bv; S.sel_i = bi;
    }
    __syncthreads();
    v_out = S.sel_d; i_out = S.sel_i;
    __syncthreads();
}

// lpc_from_cepstrum on warp 0 of the block; result in S.lpc (visible to all after the barrier)
__device__ __forceinline__ void block_lpc_from_cepstrum(const float *cep, EncScratch &S, const EncTables &T)
{
    if (threadIdx.x < 32) {
        float lpc[LPC_ORDER];
        cepstrum_to_lpc_warp(cep, S.y, S.Ex, T.dct, T.tw, T.bitrev, lpc, threadIdx.x);
        if (threadIdx.x == 0) for (int i = 0; i < LPC_ORDER; i++) S.lpc[i] = lpc[i];
    }
    __syncthreads();
}

// compute_frame_features (lpcnet_enc.c:498-577) for the frame in S.in (already pre-emphasised), sub-frame slot pc = st->pcount
__device__ void frame_features(EncState &st, EncScratch &S, const EncTables &T, int pc)
{
    const int tid = threadIdx.x;
    // aligned_in[0..80) = the tail of the previous frame (:511), analysis window (:489-493): [previous frame | this frame] x window
    if (tid < TRAINING_OFFSET_SAMPLES) S.aligned[tid] = st.analysis_mem[FRAME_SIZE - TRAINING_OFFSET_SAMPLES + tid];
    const float scale = 1.f / WINDOW_SIZE;
    for (int i = tid; i < WINDOW_SIZE; i += ENC_THREADS) {
        const float x = i < FRAME_SIZE ? st.analysis_mem[i] : S.in[i - FRAME_SIZE];
        const float w = __ldg(&T.half_window[i < FRAME_SIZE ? i : WINDOW_SIZE - 1 - i]);
        const int o = T.bitrev[i];
        S.y[o].r = scale * (x * w); S.y[o].i = scale * 0.f;       // forward_transform: x[i].i = 0 (freq.c:247), opus_fft_c scales while permuting
    }
    __syncthreads();
    if (tid < FRAME_SIZE) st.analysis_mem[tid] = S.in[tid];       // (FRAME_SIZE - OVERLAP_SIZE = 0: the whole frame is the next overlap)
    if (tid >= TRAINING_OFFSET_SAMPLES && tid < FRAME_SIZE) S.aligned[tid] = S.in[tid - TRAINING_OFFSET_SAMPLES];   // (:526)
    fft320_stages(S.y, T.tw, tid, ENC_THREADS, [] { __syncthreads(); });
    // lpcn_compute_band_energy (freq.c:131-154): band k collects frac*|X|^2 over band k-1, then (1-frac)*|X|^2 over band k, in that order
    if (tid < NB_BANDS) {
        float sum = 0;
        for (int half = 0; half < 2; half++) {
            const int b = tid - 1 + half;
            if (b < 0 || b > NB_BANDS - 2) continue;
            const int band_size = (c_eband5ms[b + 1] - c_eband5ms[b]) * 4;
            for (int j = 0; j < band_size; j++) {
                const float frac = __fdiv_rn((float)j, (float)band_size);
                const c32 X = S.y[c_eband5ms[b] * 4 + j];
                float tmp = X.r * X.r;
                tmp += X.i * X.i;
                sum += (half ? (1 - frac) : frac) * tmp;
            }
        }
        if (tid == 0 || tid == NB_BANDS - 1) sum *= 2;
        S.Ex[tid] = sum;
    }
    __syncthreads();
    if (tid == 0) {                                               // (:514-521) log spectrum with the -8 dB / -2.5 dB-per-band floors
        float logMax = -2, follow = -2;
        for (int i = 0; i < NB_BANDS; i++) {
            float ly = (float)log10(1e-2 + (double)S.Ex[i]);
            ly = MAXF(logMax - 8, MAXF(follow - 2.5f, ly));
            logMax = MAXF(logMax, ly);
            follow = MAXF(follow - 2.5f, ly);
            S.Ly[i] = ly;
        }
    }
    __syncthreads();
    if (tid < NB_BANDS) {                                         // dct (freq.c:218-228), features[0] -= 4 (:523)
        float sum = 0;
        for (int j = 0; j < NB_BANDS; j++) sum += S.Ly[j] * __ldg(&T.dct[j * NB_BANDS + tid]);
        float v = (float)((double)sum * sqrt(2. / NB_BANDS));
        if (tid == 0) v -= 4;
        st.features[pc][tid] = v;
    }
    __syncthreads();
    block_lpc_from_cepstrum(st.features[pc], S, T);               // (:524)
    if (tid < LPC_ORDER) st.features[pc][NB_BANDS + 2 + tid] = S.lpc[tid];
    // excitation history: RNN_MOVE(exc_buf, &exc_buf[FRAME_SIZE], PITCH_MAX_PERIOD) (:525)
    const float moved = st.exc_buf[FRAME_SIZE + tid];             // tid < 256 = PMAX
    __syncthreads();
    st.exc_buf[tid] = moved;
    // LPC residual (:527-537): sum = x[i] + sum_j lpc[j]*x[i-1-j] (j ascending), exc = sum + .7*previous sum
    if (tid < FRAME_SIZE) {
        float sum = S.aligned[tid];
#pragma unroll
        for (int j = 0; j < LPC_ORDER; j++) {
            const int k = tid - 1 - j;
            const float pm = k >= 0 ? S.aligned[k] : st.pitch_mem[-k - 1];
            sum += S.lpc[j] * pm;
        }
        S.sums[tid + 1] = sum;
    }
    if (tid == 0) S.sums[0] = st.pitch_filt;
    __syncthreads();
    if (tid < FRAME_SIZE) st.exc_buf[PMAX + tid] = S.sums[tid + 1] + .7f * S.sums[tid];
    if (tid < LPC_ORDER) st.pitch_mem[tid] = S.aligned[FRAME_SIZE - 1 - tid];
    if (tid == 0) st.pitch_filt = S.sums[FRAME_SIZE];
    __syncthreads();
    // cross-correlation on half-frames (:539-575)
    for (int sub = 0; sub < 2; sub++) {
        const int off = sub * FRAME_SIZE / 2;
        float *xc = st.xc[2 + 2 * pc + sub];
        {   // celt_pitch_xcorr (pitch.c:44-83): lag = tid, j ascending
            const float *x = &st.exc_buf[PMAX + off], *y = &st.exc_buf[off + tid];
            float s = 0;
            for (int j = 0; j < FRAME_SIZE / 2; j++) s = s + x[j] * y[j];
            S.xcorr[tid] = s;
        }
        if (tid == 0) {
            const float *x = &st.exc_buf[PMAX + off];
            float ener0 = 0;
            for (int j = 0; j < FRAME_SIZE / 2; j++) ener0 = ener0 + x[j] * x[j];
            st.frame_weight[2 + 2 * pc + sub] = ener0;
            const float *e = &st.exc_buf[off];
            float ip = 0;
            for (int j = 0; j < FRAME_SIZE / 2 - 1; j++) ip = ip + e[j] * e[j];
            double ener1 = ip;                                    // `double ener1` (:541): the sliding energy is updated in double
            for (int i = 0; i < PMAX; i++) {
                ener1 += e[i + FRAME_SIZE / 2 - 1] * e[i + FRAME_SIZE / 2 - 1];
                S.en[i] = (float)((double)(1 + ener0) + ener1);
                ener1 -= e[i] * e[i];
            }
        }
        __syncthreads();
        xc[tid] = __fdiv_rn(2 * S.xcorr[tid], S.en[tid]);
        __syncthreads();
        // upsample the correlation by 3 and keep the maximum (:556-571)
        if (tid >= 4 && tid < PMAX - 4) {
            const float interp[7] = {0.026184f, -0.098339f, 0.369938f, 0.837891f, -0.184969f, 0.070242f, -0.020947f};
            float val1 = 0, val2 = 0;
            for (int j = 0; j < 7; j++) { val1 += xc[tid - 3 + j] * interp[j]; val2 += xc[tid + 3 - j] * interp[j]; }
            S.tmp[tid] = MAXF(xc[tid], MAXF(val1, val2));
        }
        __syncthreads();
        if (tid >= 4 && tid < PMAX - 4) xc[tid] = S.tmp[tid];
        __syncthreads();
    }
}

// one forward step of the pitch Viterbi search over sub-frame row `row` (lpcnet_enc.c:603-634 / :828-859), back pointers into pp[]
__device__ void viterbi_step(EncState &st, EncScratch &S, int row, unsigned char *pp)
{
    const int tid = threadIdx.x;
    float *xc = st.xc[row];
    const float w = st.frame_weight[row];
    // sub-harmonic attenuation (:606-609): every read is of a not-yet-modified entry ((PMAX+i-1)/2 > i for i < 192)
    float att = 0; bool do_att = false;
    if (tid < PMAX - 2 * PMIN) {
        const float xc_half = MAXF(MAXF(xc[(PMAX + tid) / 2], xc[(PMAX + tid + 2) / 2]), xc[(PMAX + tid - 1) / 2]);
        if (xc[tid] < xc_half * 1.1f) { do_att = true; att = xc[tid] * .8f; }
    }
    __syncthreads();
    if (do_att) xc[tid] = att;
    __syncthreads();
    float mine = -3e38f;
    if (tid < PMAX - PMIN) {
        float max_prev = st.pmp_all - 6.f;
        int prev = st.best_i;
        const int jlo = -4 > -tid ? -4 : -tid;
        for (int j = jlo; j <= 4 && tid + j < PMAX - PMIN; j++) {
            const int aj = j < 0 ? -j : j;
            const float cand = st.pmp[0][tid + j] - .02f * aj * aj;
            if (cand > max_prev) { max_prev = cand; prev = tid + j; }
        }
        pp[tid] = (unsigned char)prev;
        mine = max_prev + w * xc[tid];
        st.pmp[1][tid] = mine;
    }
    float max_all; int best;
    block_argmax(mine, tid, S, max_all, best);                    // (`> max_path_all` from -1e15: the first maximum wins)
    if (tid < PMAX - PMIN) st.pmp[1][tid] -= max_all;             // renormalise (:631)
    __syncthreads();
    st.pmp[0][tid] = st.pmp[1][tid];                              // RNN_COPY of all PITCH_MAX_PERIOD entries (:634)
    if (tid == 0) { st.pmp_all = max_all; st.best_i = best; }
    __syncthreads();
}

// process_single_frame (lpcnet_enc.c:814-870)
__device__ void single_frame(EncState &st, EncScratch &S, int pc)
{
    const int tid = threadIdx.x;
    if (tid == 0) {
        float s = 1e-15f;
        for (int sub = 0; sub < 2; sub++) s += st.frame_weight[2 + 2 * pc + sub];
        for (int sub = 0; sub < 2; sub++) st.frame_weight[2 + 2 * pc + sub] *= (2.f / s);
    }
    __syncthreads();
    for (int sub = 0; sub < 2; sub++) viterbi_step(st, S, 2 + 2 * pc + sub, S.pitch_prev[sub]);
    if (tid == 0) {
        int best_i = st.best_i, best[4];
        float frame_corr = 0;
        for (int sub = 1; sub >= 0; sub--) {
            best[2 + sub] = PMAX - best_i;
            frame_corr += st.frame_weight[2 + 2 * pc + sub] * st.xc[2 + 2 * pc + sub][best_i];
            best_i = S.pitch_prev[sub][best_i];
        }
        frame_corr /= 2;
        int b = best[2] + best[3];
        b = b < 510 ? b : 510; b = b > 66 ? b : 66;
        st.features[pc][NB_BANDS] = .01f * (b - 200);
        st.features[pc][NB_BANDS + 1] = frame_corr - .5f;
    }
    __syncthreads();
}

// vq_quantize_mbest (lpcnet_enc.c:53-78) with mbest = 5 over 1024 entries of 17 dims: = the five smallest (distance, index) pairs
__device__ void vq_mbest5(const float *cb, const float *x, EncScratch &S, float *dist, int *index)
{
    const int tid = threadIdx.x;
    float d[4]; bool taken[4];
#pragma unroll
    for (int e = 0; e < 4; e++) {
        const int i = tid + e * ENC_THREADS;
        float acc = 0;
        for (int j = 0; j < NB_BANDS - 1; j++) { const float df = x[j] - __ldg(&cb[i * (NB_BANDS - 1) + j]); acc += df * df; }
        d[e] = acc; taken[e] = false;
    }
    for (int m = 0; m < 5; m++) {
        float bd = 3e38f; int bi = 0x7fffffff;
#pragma unroll
        for (int e = 0; e < 4; e++) if (!taken[e] && (d[e] < bd)) { bd = d[e]; bi = tid + e * ENC_THREADS; }
        float gd; int gi;
        block_argmin(bd, bi, S, gd, gi);
#pragma unroll
        for (int e = 0; e < 4; e++) if (gi == tid + e * ENC_THREADS) taken[e] = true;
        if (tid == 0) { dist[m] = gd; index[m] = gi; }
    }
    __syncthreads();
}

struct Quant { int c0_id, vq_end[3], vq_mid, interp_id; };

// the quantisation block of process_superframe (lpcnet_enc.c:700-711)
__device__ void quantize_superframe(EncState &st, EncScratch &S, const EncTables &T, Quant &q)
{
    const int tid = threadIdx.x;
    const float *cb1 = T.cb, *cb2 = cb1 + 1024 * 17, *cb3 = cb2 + 1024 * 17, *cbd = cb3 + 1024 * 17;
    __shared__ float cur_d[5], glob_d[5]; __shared__ int cur_i[5], idx1[5], idx2[5][2], idx3[5][3];
    __shared__ float diff[NB_BANDS];
    __shared__ int s_c0, s_mid, s_interp;
    if (tid == 0) {
        int c0 = cvtt_x86(floor(.5 + (double)(st.features[3][0] * 4)));
        c0 = c0 < 63 ? c0 : 63; c0 = c0 > -64 ? c0 : -64;
        st.features[3][0] = c0 / 4.f;
        s_c0 = c0;
    }
    __syncthreads();
    // ---- quantize_3stage_mbest(&features[3][1], vq_end) (:133-241) ----
    float *x = &st.features[3][1];
    vq_mbest5(cb1, x, S, cur_d, cur_i);
    if (tid < 5) idx1[tid] = cur_i[tid];
    __syncthreads();
    for (int k = 0; k < 5; k++) {
        if (tid < NB_BANDS - 1) diff[tid] = x[tid] - __ldg(&cb1[idx1[k] * 17 + tid]);
        __syncthreads();
        vq_mbest5(cb2, diff, S, cur_d, cur_i);
        if (tid == 0) {
            if (k == 0) { for (int m = 0; m < 5; m++) { idx2[m][0] = idx1[k]; idx2[m][1] = cur_i[m]; glob_d[m] = cur_d[m]; } }
            else if (cur_d[0] < glob_d[4]) {
                int m = 0;
                for (int pos = 0; pos < 5; pos++) {
                    if (cur_d[m] < glob_d[pos]) {
                        for (int j = 4; j >= pos + 1; j--) { glob_d[j] = glob_d[j - 1]; idx2[j][0] = idx2[j - 1][0]; idx2[j][1] = idx2[j - 1][1]; }
                        glob_d[pos] = cur_d[m]; idx2[pos][0] = idx1[k]; idx2[pos][1] = cur_i[m];
                        m++;
                    }
                }
            }
        }
        __syncthreads();
    }
    for (int k = 0; k < 5; k++) {
        if (tid < NB_BANDS - 1) diff[tid] = x[tid] - __ldg(&cb1[idx2[k][0] * 17 + tid]) - __ldg(&cb2[idx2[k][1] * 17 + tid]);
        __syncthreads();
        vq_mbest5(cb3, diff, S, cur_d, cur_i);
        if (tid == 0) {
            if (k == 0) { for (int m = 0; m < 5; m++) { idx3[m][0] = idx2[k][0]; idx3[m][1] = idx2[k][1]; idx3[m][2] = cur_i[m]; glob_d[m] = cur_d[m]; } }
            else if (cur_d[0] < glob_d[4]) {
                int m = 0;
                for (int pos = 0; pos < 5; pos++) {
                    if (cur_d[m] < glob_d[pos]) {
                        for (int j = 4; j >= pos + 1; j--) { glob_d[j] = glob_d[j - 1]; idx3[j][0] = idx3[j - 1][0]; idx3[j][1] = idx3[j - 1][1]; idx3[j][2] = idx3[j - 1][2]; }
                        glob_d[pos] = cur_d[m]; idx3[pos][0] = idx2[k][0]; idx3[pos][1] = idx2[k][1]; idx3[pos][2] = cur_i[m];
                        m++;
                    }
                }
            }
        }
        __syncthreads();
    }
    const int id = idx3[0][0], id2 = idx3[0][1], id3 = idx3[0][2];
    if (tid < NB_BANDS - 1) x[tid] = __ldg(&cb1[id * 17 + tid]) + __ldg(&cb2[id2 * 17 + tid]) + __ldg(&cb3[id3 * 17 + tid]);   // (:227-229)
    __syncthreads();
    // ---- quantize_diff(features[1], vq_mem, features[3], ceps_codebook_diff4, 12, 1, &vq_mid) (:283-318) ----
    {
        float *xm = st.features[1]; const float *left = st.vq_mem, *right = st.features[3];
        if (tid < NB_BANDS) {
            const float p = .5f * (left[tid] + right[tid]);
            S.vq_pred[tid] = p; S.vq_pred[NB_BANDS + tid] = p; S.vq_pred[2 * NB_BANDS + tid] = left[tid]; S.vq_pred[3 * NB_BANDS + tid] = right[tid];
        }
        __syncthreads();
        if (tid < 4 * NB_BANDS) S.vq_target[tid] = xm[tid % NB_BANDS] - S.vq_pred[tid];
        __syncthreads();
        // find_nearest_multi (:243-280): entries i (difference) in order, then the negated entries as i + 4096; first minimum wins
        float bd = 3e38f; int bi = 0x7fffffff;
        for (int sgn = 0; sgn < 2; sgn++)
            for (int e = 0; e < 4096 / ENC_THREADS; e++) {
                const int i = tid + e * ENC_THREADS;
                const float *tg = &S.vq_target[(i & 3) * NB_BANDS];
                float acc = 0;
                for (int j = 0; j < NB_BANDS; j++) {
                    const float c = __ldg(&cbd[i * NB_BANDS + j]);
                    const float df = sgn ? tg[j] + c : tg[j] - c;
                    acc += df * df;
                }
                const int ci = i + sgn * 4096;
                if (acc < bd || (acc == bd && ci < bi)) { bd = acc; bi = ci; }
            }
        float gd; int gi;
        block_argmin(bd, bi, S, gd, gi);
        int idd = gi; float sg = 1;
        if (idd >= 4096) { sg = -1; idd -= 4096; }
        if (tid == 0) s_mid = gi;
        if (tid < NB_BANDS) xm[tid] = S.vq_pred[(idd & 3) * NB_BANDS + tid] + sg * __ldg(&cbd[idd * NB_BANDS + tid]);
        __syncthreads();
    }
    // ---- double_interp_search (:379-401) + perform_double_interp (common.c:58-65) ----
    if (tid == 0) {
        float dist[2][3];
        for (int h = 0; h < 2; h++) {       // interp_search(features[0], mem, features[1]) / (features[2], features[1], features[3]) (:320-341)
            const float *xx = st.features[2 * h], *left = h ? st.features[1] : st.vq_mem, *right = st.features[2 * h + 1];
            for (int k = 1; k < 4; k++) {
                float dd = 0;
                for (int i = 0; i < NB_BANDS; i++) {
                    const float p = k == 1 ? .5f * (left[i] + right[i]) : (k == 2 ? left[i] : right[i]);
                    dd += (xx[i] - p) * (xx[i] - p);
                }
                dist[h][k - 1] = dd;
            }
        }
        int best_id = 0; float min_dist = 1e15f;
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
            const int idn = 3 * i + j; const float dd = dist[0][i] + dist[1][j];
            if (dd < min_dist && idn != 7) { min_dist = dd; best_id = idn; }
        }
        s_interp = best_id - (best_id >= 7);
    }
    __syncthreads();
    {
        int bid = s_interp; bid += (bid >= 7);
        const int id0 = bid / 3, id1 = bid % 3;
        float v0 = 0, v2 = 0;
        if (tid < NB_BANDS) {     // single_interp reads left/right before anything is written: features[1] and [3] are not modified here
            const float l0 = st.vq_mem[tid], r0 = st.features[1][tid], l1 = st.features[1][tid], r1 = st.features[3][tid];
            v0 = id0 == 0 ? .5f * (l0 + r0) : (id0 == 1 ? l0 : r0);
            v2 = id1 == 0 ? .5f * (l1 + r1) : (id1 == 1 ? l1 : r1);
        }
        __syncthreads();
        if (tid < NB_BANDS) { st.features[0][tid] = v0; st.features[2][tid] = v2; }
    }
    __syncthreads();
    q.c0_id = s_c0; q.vq_end[0] = id; q.vq_end[1] = id2; q.vq_end[2] = id3; q.vq_mid = s_mid; q.interp_id = s_interp;
}

// process_superframe (lpcnet_enc.c:579-744) after four compute_frame_features calls
__device__ void superframe(EncState &st, EncScratch &S, const EncTables &T, bool quantize, unsigned char *packet)
{
    const int tid = threadIdx.x;
    __shared__ int s_main_pitch, s_modulation, s_corr_id, s_voiced;
    if (tid == 0) {
        float s = 1e-15f;
        for (int sub = 0; sub < 8; sub++) s += st.frame_weight[2 + sub];
        for (int sub = 0; sub < 8; sub++) st.frame_weight[2 + sub] *= (8.f / s);
    }
    __syncthreads();
    for (int sub = 0; sub < 8; sub++) viterbi_step(st, S, 2 + sub, S.pitch_prev[sub]);
    if (tid == 0) {
        int best_i = st.best_i; int *best = S.best;
        float frame_corr = 0;
        for (int sub = 7; sub >= 0; sub--) {
            best[2 + sub] = PMAX - best_i;
            frame_corr += st.frame_weight[2 + sub] * st.xc[2 + sub][best_i];
            best_i = S.pitch_prev[sub][best_i];
        }
        frame_corr /= 8;
        if (quantize && frame_corr < 0) frame_corr = 0;
        float sx = 0, sxx = 0, sxy = 0, sy = 0, sw = 0;
        for (int sub = 2; sub < 10; sub++) {
            const float w = st.frame_weight[sub];
            sw += w; sx += w * sub; sxx += w * sub * sub; sxy += w * sub * best[sub]; sy += w * best[sub];
        }
        const int voiced = (double)frame_corr >= .3;
        float best_a = (sw * sxy - sx * sy) / (sw * sxx - sx * sx);
        int corr_id;
        if (voiced) {
            const float mean_pitch = sy / sw, max_a = mean_pitch / 32;
            best_a = MINF(max_a, MAXF(-max_a, best_a));
            corr_id = cvtt_x86(floor((double)((frame_corr - .3f) / .175f)));
            if (quantize) frame_corr = 0.3875f + .175f * corr_id;
        } else {
            best_a = 0;
            corr_id = cvtt_x86(floor((double)(frame_corr / .075f)));
            if (quantize) frame_corr = 0.0375f + .075f * corr_id;
        }
        const float best_b = (sy - best_a * sx) / sw;
        const float center_pitch = best_b + 5.5f * best_a;
        // a superframe with excitation energy in one half-subframe only can make the slope 0/0: best_a and center_pitch are then
        // NaN and the conversions must give INT_MIN like the reference's (modulation -3, packet field 1), not CUDA's 0
        int main_pitch = cvtt_x86(floor(.5 + 21. * 1.442695041 * log((double)(center_pitch / PMIN))));
        main_pitch = main_pitch < 63 ? main_pitch : 63; main_pitch = main_pitch > 0 ? main_pitch : 0;
        int modulation = cvtt_x86(floor(.5 + (double)(16 * 7 * best_a / center_pitch)));
        modulation = modulation < 3 ? modulation : 3; modulation = modulation > -3 ? modulation : -3;
        for (int sub = 0; sub < 4; sub++) {
            if (quantize) {
                float p = __ldg(&T.pitch_pow[main_pitch]);                     // (float)(pow(2.f, main_pitch/21.)*PITCH_MIN_PERIOD), host-built
                p *= 1.f + modulation / 16.f / 7.f * (2 * sub - 3);
                p = MINF(255, MAXF(33, p));
                st.features[sub][NB_BANDS] = .02f * (p - 100);
            } else {
                int b = best[2 + 2 * sub] + best[2 + 2 * sub + 1];
                b = b < 510 ? b : 510; b = b > 66 ? b : 66;
                st.features[sub][NB_BANDS] = .01f * (b - 200);
            }
            st.features[sub][NB_BANDS + 1] = frame_corr - .5f;
        }
        s_main_pitch = main_pitch; s_modulation = modulation; s_corr_id = corr_id; s_voiced = voiced;
    }
    __syncthreads();
    st.xc[0][tid] = st.xc[8][tid]; st.xc[1][tid] = st.xc[9][tid];                 // (:697-698)
    __syncthreads();
    Quant q = {0, {0, 0, 0}, 0, 0};
    if (quantize) quantize_superframe(st, S, T, q);
    for (int sub = 0; sub < 4; sub++) {                                            // (:714-717)
        block_lpc_from_cepstrum(st.features[sub], S, T);
        if (tid < LPC_ORDER) st.features[sub][NB_BANDS + 2 + tid] = S.lpc[tid];
        __syncthreads();
    }
    if (tid < NB_BANDS) st.vq_mem[tid] = st.features[3][tid];
    if (packet && tid == 0) {                                                      // bits_pack, MSB first (:443-463, :724-733)
        unsigned long long bits = 0; int pos = 0;
        auto put = [&](unsigned v, int nb) { bits |= (unsigned long long)(v & ((1u << nb) - 1)) << (64 - pos - nb); pos += nb; };
        put((unsigned)(q.c0_id + 64), 7); put((unsigned)s_main_pitch, 6); put((unsigned)(s_voiced ? s_modulation + 4 : 0), 3); put((unsigned)s_corr_id, 2);
        put((unsigned)q.vq_end[0], 10); put((unsigned)q.vq_end[1], 10); put((unsigned)q.vq_end[2], 10); put((unsigned)q.vq_mid, 13); put((unsigned)q.interp_id, 3);
        for (int i = 0; i < 8; i++) packet[i] = (unsigned char)(bits >> (56 - 8 * i));
    }
    __syncthreads();
}

// MODE 0: lpcnet_compute_single_frame_features per frame; 1: lpcnet_encode per packet; 2: lpcnet_compute_features per packet
template <int MODE>
__global__ void __launch_bounds__(ENC_THREADS, 4) enc_kernel(const EncArgs a)
{
    __shared__ EncState st;
    __shared__ EncScratch S;
    const int s = blockIdx.x, tid = threadIdx.x;
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(a.state + s);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&st);
        for (int i = tid; i < ENC_STATE_WORDS; i += ENC_THREADS) dst[i] = src[i];
    }
    __syncthreads();
    const int fpu = MODE == 0 ? 1 : 4;                               // frames per unit
    for (int u = 0; u < a.units; u++) {
        for (int k = 0; k < fpu; k++) {
            // pcm -> float, preemphasis (lpcnet_enc.c:872-880): y[i] = x[i] + mem, mem = -coef*x[i]
            const size_t base = ((size_t)s * a.units + u) * fpu * FRAME_SIZE + (size_t)k * FRAME_SIZE;
            if (tid < FRAME_SIZE) {
                const float xi = a.pcm16 ? (float)a.pcm16[base + tid] : a.pcmf[base + tid];
                float mem;
                if (tid == 0) mem = st.mem_preemph;
                else { const float xp = a.pcm16 ? (float)a.pcm16[base + tid - 1] : a.pcmf[base + tid - 1]; mem = -0.85f * xp; }
                S.in[tid] = xi + mem;
                if (tid == FRAME_SIZE - 1) S.sums[0] = -0.85f * xi;  // next mem_preemph (parked until the barrier)
            }
            __syncthreads();
            if (tid == 0) { st.mem_preemph = S.sums[0]; if (MODE != 0) st.pcount = k; }
            __syncthreads();
            const int pc = st.pcount;
            frame_features(st, S, a.t, pc);
            if (MODE == 0) {
                single_frame(st, S, pc);
                if (tid < NTOT) a.features[((size_t)s * a.units + u) * NTOT + tid] = st.features[0][tid];   // RNN_COPY(features, &st->features[0][0]) (:915)
                __syncthreads();
            }
        }
        if (MODE == 1) superframe(st, S, a.t, true, a.packets + ((size_t)s * a.units + u) * 8);
        if (MODE == 2) {
            superframe(st, S, a.t, false, nullptr);
            if (tid < 4 * NTOT) a.features[((size_t)s * a.units + u) * 4 * NTOT + tid] = st.features[tid / NTOT][tid % NTOT];
            __syncthreads();
        }
    }
    {
        uint32_t *dst = reinterpret_cast<uint32_t *>(a.state + s);
        const uint32_t *src = reinterpret_cast<const uint32_t *>(&st);
        for (int i = tid; i < ENC_STATE_WORDS; i += ENC_THREADS) dst[i] = src[i];
    }
}

}  // namespace lpcnet_b200

// ---------------------------------------------------------------------------------------------------------------------------
using namespace lpcnet_b200;

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_error("%s failed: %s", #call, cudaGetErrorString(e_)); return -1; } } while (0)

struct LPCNetB200EncBatch {
    int device, n;
    EncState *state;
    float *half_window, *dct, *twiddles, *pitch_pow, *cb;
    int16_t *bitrev;
    void *d_in; size_t d_in_cap;
    void *d_out; size_t d_out_cap;
    cudaStream_t stream;
    // Ordering of the encoder state across CUDA streams, as in LPCNetB200Batch: every call that enqueues work records `order_ev`
    // on the stream it used and the next call makes ITS stream wait for that event first, so consecutive `_device` calls may
    // use different streams and may be mixed with the host-pointer calls.
    cudaEvent_t order_ev; cudaStream_t last_stream; bool has_order;
};

namespace lpcnet_b200 { void build_fft_tables(std::vector<float> &dct, std::vector<float> &tw, std::vector<int16_t> &br); }

static int enc_order_enter(LPCNetB200EncBatch *e, cudaStream_t st)
{
    if (e->has_order && e->last_stream != st) CK(cudaStreamWaitEvent(st, e->order_ev, 0));
    return 0;
}
static int enc_order_leave(LPCNetB200EncBatch *e, cudaStream_t st)
{
    CK(cudaEventRecord(e->order_ev, st));
    e->last_stream = st; e->has_order = true;
    return 0;
}

static int enc_grow(void **p, size_t *cap, size_t bytes)
{
    if (*cap >= bytes) return 0;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    CK(cudaMalloc(p, bytes));
    *cap = bytes;
    return 0;
}

extern "C" {

void lpcnet_b200_enc_destroy(LPCNetB200EncBatch *e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    void *ptrs[] = {e->state, e->half_window, e->dct, e->twiddles, e->pitch_pow, e->cb, e->bitrev, e->d_in, e->d_out};
    if (e->order_ev) { if (e->has_order) cudaEventSynchronize(e->order_ev); cudaEventDestroy(e->order_ev); }
    for (void *p : ptrs) if (p) cudaFree(p);
    if (e->stream) cudaStreamDestroy(e->stream);
    free(e);
}

int lpcnet_b200_enc_reset(LPCNetB200EncBatch *e)
{
    if (!e) { set_error("null encoder batch"); return -1; }
    CK(cudaSetDevice(e->device));
    if (enc_order_enter(e, e->stream)) return -1;
    CK(cudaMemsetAsync(e->state, 0, sizeof(EncState) * (size_t)e->n, e->stream));    // lpcnet_encoder_init: memset(st, 0) (lpcnet_enc.c:471-475)
    if (enc_order_leave(e, e->stream)) return -1;
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

// half_window / dct_table exactly as src/dump_lpcnet_tables.c:83-96 generates them (double math, stored as float)
void lpcnet_b200_enc_tables(float *half_window, float *dct)
{
    for (int i = 0; i < FRAME_SIZE; i++) half_window[i] = (float)sin(.5 * M_PI * sin(.5 * M_PI * (i + .5) / FRAME_SIZE) * sin(.5 * M_PI * (i + .5) / FRAME_SIZE));
    for (int i = 0; i < NB_BANDS; i++) for (int j = 0; j < NB_BANDS; j++) {
        double v = cos((i + .5) * j * M_PI / NB_BANDS);
        if (j == 0) v *= sqrt(.5);
        dct[i * NB_BANDS + j] = (float)v;
    }
}

LPCNetB200EncBatch *lpcnet_b200_enc_create(int n_streams, int device)
{
    if (n_streams <= 0) { set_error("n_streams must be positive"); return nullptr; }
    const int cnt = lpcnet_b200_device_count();
    if (cnt <= 0) { set_error("no CUDA device available (this engine has no CPU fallback)"); return nullptr; }
    if (device < 0 || device >= cnt) { set_error("device %d out of range (%d devices)", device, cnt); return nullptr; }
    if (cudaSetDevice(device) != cudaSuccess) { set_error("cudaSetDevice(%d) failed", device); return nullptr; }
    LPCNetB200EncBatch *e = (LPCNetB200EncBatch *)calloc(1, sizeof(*e));
    e->device = device; e->n = n_streams;
    std::vector<float> hw(FRAME_SIZE), dct, tw, pp(64);
    std::vector<int16_t> br;
    build_fft_tables(dct, tw, br);
    std::vector<float> dct2(NB_BANDS * NB_BANDS);
    lpcnet_b200_enc_tables(hw.data(), dct2.data());
    for (int k = 0; k < 64; k++) pp[k] = (float)(pow(2.f, k / 21.) * 32);                 // lpcnet_enc.c:684 / lpcnet_dec.c:124
    bool ok = true;
    auto up = [&](void **dst, const void *src, size_t bytes) { if (ok && (cudaMalloc(dst, bytes) != cudaSuccess || cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess)) ok = false; };
    up((void **)&e->half_window, hw.data(), hw.size() * 4); up((void **)&e->dct, dct2.data(), dct2.size() * 4);
    up((void **)&e->twiddles, tw.data(), tw.size() * 4); up((void **)&e->bitrev, br.data(), br.size() * 2); up((void **)&e->pitch_pow, pp.data(), pp.size() * 4);
    if (ok && cudaMalloc((void **)&e->state, sizeof(EncState) * (size_t)n_streams) != cudaSuccess) ok = false;
    if (ok && cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) ok = false;
    if (ok && cudaEventCreateWithFlags(&e->order_ev, cudaEventDisableTiming) != cudaSuccess) ok = false;
    if (!ok || lpcnet_b200_enc_reset(e) != 0) { set_error("encoder batch: device allocation failed: %s", cudaGetErrorString(cudaGetLastError())); lpcnet_b200_enc_destroy(e); return nullptr; }
    return e;
}

int lpcnet_b200_enc_streams(const LPCNetB200EncBatch *e) { return e ? e->n : 0; }

int lpcnet_b200_enc_set_codebooks(LPCNetB200EncBatch *e, const float *cb, size_t n_floats)
{
    if (!e) { set_error("null encoder batch"); return -1; }
    const size_t want = 3 * 1024 * 17 + 4096 * 18;
    if (!cb || n_floats != want) { set_error("codebooks: expected %zu floats", want); return -1; }
    CK(cudaSetDevice(e->device));
    if (!e->cb) CK(cudaMalloc((void **)&e->cb, want * sizeof(float)));
    CK(cudaMemcpy(e->cb, cb, want * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// mode 0: features per frame, 1: packets, 2: features per 4-frame packet; input on the device
static int enc_run_device(LPCNetB200EncBatch *e, int mode, const short *d_pcm16, const float *d_pcmf, int units, float *d_features, unsigned char *d_packets, cudaStream_t st)
{
    if (units <= 0) return 0;
    if (mode == 1 && !e->cb) { set_error("encode: no VQ codebooks loaded (lpcnet_b200_enc_set_codebooks)"); return -1; }
    EncArgs a{e->state, e->n, d_pcm16, d_pcmf, units, d_features, d_packets,
              EncTables{e->half_window, e->dct, reinterpret_cast<const c32 *>(e->twiddles), e->bitrev, e->pitch_pow, e->cb}};
    if (enc_order_enter(e, st)) return -1;
    if (mode == 0) enc_kernel<0><<<e->n, ENC_THREADS, 0, st>>>(a);
    else if (mode == 1) enc_kernel<1><<<e->n, ENC_THREADS, 0, st>>>(a);
    else enc_kernel<2><<<e->n, ENC_THREADS, 0, st>>>(a);
    CK(cudaGetLastError());
    return enc_order_leave(e, st);
}

static int enc_run_host(LPCNetB200EncBatch *e, int mode, const void *pcm, bool is_float, int units, float *features, unsigned char *packets)
{
    if (!e) { set_error("null encoder batch"); return -1; }
    if (units <= 0) return 0;
    if (!pcm || (mode == 1 ? !packets : !features)) { set_error("null buffer"); return -1; }
    CK(cudaSetDevice(e->device));
    const size_t samples = (size_t)e->n * units * (mode == 0 ? FRAME_SIZE : 4 * FRAME_SIZE);
    const size_t ibytes = samples * (is_float ? 4 : 2);
    const size_t obytes = mode == 1 ? (size_t)e->n * units * 8 : (size_t)e->n * units * (mode == 0 ? 1 : 4) * NTOT * sizeof(float);
    CK(cudaStreamSynchronize(e->stream));
    if (enc_grow(&e->d_in, &e->d_in_cap, ibytes) || enc_grow(&e->d_out, &e->d_out_cap, obytes)) return -1;
    CK(cudaMemcpyAsync(e->d_in, pcm, ibytes, cudaMemcpyHostToDevice, e->stream));
    if (enc_run_device(e, mode, is_float ? nullptr : (const short *)e->d_in, is_float ? (const float *)e->d_in : nullptr, units,
                       mode == 1 ? nullptr : (float *)e->d_out, mode == 1 ? (unsigned char *)e->d_out : nullptr, e->stream)) return -1;
    CK(cudaMemcpyAsync(mode == 1 ? (void *)packets : (void *)features, e->d_out, obytes, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

int lpcnet_b200_enc_compute_features(LPCNetB200EncBatch *e, const short *pcm, int nframes, float *features) { return enc_run_host(e, 0, pcm, false, nframes, features, nullptr); }
int lpcnet_b200_enc_compute_features_float(LPCNetB200EncBatch *e, const float *pcm, int nframes, float *features) { return enc_run_host(e, 0, pcm, true, nframes, features, nullptr); }
int lpcnet_b200_enc_encode(LPCNetB200EncBatch *e, const short *pcm, int npackets, unsigned char *packets) { return enc_run_host(e, 1, pcm, false, npackets, nullptr, packets); }
int lpcnet_b200_enc_compute_features4(LPCNetB200EncBatch *e, const short *pcm, int npackets, float *features) { return enc_run_host(e, 2, pcm, false, npackets, features, nullptr); }

int lpcnet_b200_enc_compute_features_device(LPCNetB200EncBatch *e, const short *d_pcm, int nframes, float *d_features, void *cuda_stream)
{
    if (!e || !d_pcm || !d_features) { set_error("enc_compute_features_device: null argument"); return -1; }
    CK(cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    if (enc_run_device(e, 0, d_pcm, nullptr, nframes, d_features, nullptr, st)) return -1;
    if (!cuda_stream) CK(cudaStreamSynchronize(st));
    return 0;
}
int lpcnet_b200_enc_encode_device(LPCNetB200EncBatch *e, const short *d_pcm, int npackets, unsigned char *d_packets, void *cuda_stream)
{
    if (!e || !d_pcm || !d_packets) { set_error("enc_encode_device: null argument"); return -1; }
    CK(cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    if (enc_run_device(e, 1, d_pcm, nullptr, npackets, nullptr, d_packets, st)) return -1;
    if (!cuda_stream) CK(cudaStreamSynchronize(st));
    return 0;
}

}  // extern "C"
