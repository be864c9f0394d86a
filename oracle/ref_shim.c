/* TEST INFRASTRUCTURE — compiled together with the untouched reference sources (oracle/Makefile `ref`).
 * Gives the Python tests a few convenience entry points around the reference's own public API
 * (include/lpcnet.h) and exposes static-inline helpers of the reference (common.h, vec_avx.h) by value.
 * Nothing here re-implements reference behaviour. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <immintrin.h>
#include "nnet_data.h"
#include "nnet.h"
#include "common.h"
#include "freq.h"
#include "lpcnet.h"
#include "lpcnet_private.h"

/* _mm_rcp_ss on mantissa bin k (top 11 mantissa bits), exponent 0: the table the engine must emulate. */
void ref_rcp_table(uint32_t *out)
{
    int k;
    for (k = 0; k < 2048; k++) {
        union { float f; uint32_t u; } in, o;
        in.u = 0x3f800000u | ((uint32_t)k << 12);
        o.f = _mm_cvtss_f32(_mm_rcp_ss(_mm_set_ss(in.f)));
        out[k] = o.u;
    }
}

float ref_rcp(float x) { return _mm_cvtss_f32(_mm_rcp_ss(_mm_set_ss(x))); }
/* _mm256_rcp_ps (the instruction inside tanh8_approx / sigmoid8_approx, vec_avx.h:408,437) on n floats */
void ref_rcp8(const float *x, float *out, int n)
{
    int i, j;
    for (i = 0; i < n; i += 8) {
        float in[8] = {0}, o[8];
        for (j = 0; j < 8 && i + j < n; j++) in[j] = x[i + j];
        _mm256_storeu_ps(o, _mm256_rcp_ps(_mm256_loadu_ps(in)));
        for (j = 0; j < 8 && i + j < n; j++) out[i + j] = o[j];
    }
}
int ref_lin2ulaw(float x) { return lin2ulaw(x); }
float ref_ulaw2lin(float u) { return ulaw2lin(u); }
void ref_activation(float *out, const float *in, int n, int act) { compute_activation(out, in, n, act); }
int ref_state_size(void) { return lpcnet_get_size(); }
int ref_is_float_build(void)
{
#ifdef DOT_PROD
    return 0;
#else
    return 1;
#endif
}

/* Synthesise nframes frames (features: [nframes][stride] floats, first 20 used) with a fresh state.  blob NULL: keep the
 * model lpcnet_create() set up, i.e. the arrays compiled in from nnet_data.c (a build without USE_WEIGHTS_FILE). */
int ref_synth_stream(const unsigned char *blob, int len, const float *features, int stride, int nframes,
                     short *pcm)
{
    int i;
    LPCNetState *st = lpcnet_create();
    if (blob && lpcnet_load_model(st, blob, len) != 0) { lpcnet_destroy(st); return -1; }
    for (i = 0; i < nframes; i++)
        lpcnet_synthesize(st, features + (size_t)i * stride, pcm + (size_t)i * LPCNET_FRAME_SIZE, LPCNET_FRAME_SIZE);
    lpcnet_destroy(st);
    return 0;
}

/* Decode npackets 8-byte packets with a fresh decoder state. LPCNetDecState starts with its LPCNetState
 * (lpcnet_private.h:50-53) so the blob is loaded through that member; blob NULL: the compiled-in arrays, as above. */
int ref_decode_stream(const unsigned char *blob, int len, const unsigned char *packets, int npackets, short *pcm)
{
    int i;
    LPCNetDecState *st = lpcnet_decoder_create();
    if (blob && lpcnet_load_model((LPCNetState *)st, blob, len) != 0) { lpcnet_decoder_destroy(st); return -1; }
    for (i = 0; i < npackets; i++)
        lpcnet_decode(st, packets + (size_t)i * LPCNET_COMPRESSED_SIZE, pcm + (size_t)i * LPCNET_PACKET_SAMPLES);
    lpcnet_decoder_destroy(st);
    return 0;
}

void ref_decode_packet(float *features /*[4][36]*/, float *vq_mem /*[18]*/, const unsigned char *buf)
{
    decode_packet((float (*)[NB_TOTAL_FEATURES])features, vq_mem, buf);
}

/* One call of the reference frame network on a fresh state after `warm` warm-up frames: dumps conditioning + lpc. */
int ref_frame_network(const unsigned char *blob, int len, const float *features, int stride, int nframes,
                      float *gru_a_cond /*[nframes][1152]*/, float *gru_b_cond /*[nframes][48]*/, float *lpc /*[nframes][16]*/)
{
    int i;
    LPCNetState *st = lpcnet_create();
    if (lpcnet_load_model(st, blob, len) != 0) { lpcnet_destroy(st); return -1; }
    for (i = 0; i < nframes; i++)
        run_frame_network(st, gru_a_cond + (size_t)i * 3 * GRU_A_STATE_SIZE, gru_b_cond + (size_t)i * 3 * GRU_B_STATE_SIZE,
                          lpc + (size_t)i * LPC_ORDER, features + (size_t)i * stride);
    lpcnet_destroy(st);
    return 0;
}

/* ---- the internal entry points the reference's PLC uses (lpcnet_private.h:125-133) on an explicit state handle, so that the
 * tests can drive the same call sequence on the reference, the oracle port and the engine ---- */
void *ref_state_create(const unsigned char *blob, int len)
{
    LPCNetState *st = lpcnet_create();
    if (lpcnet_load_model(st, blob, len) != 0) { lpcnet_destroy(st); return NULL; }
    return st;
}
void ref_state_destroy(void *st) { lpcnet_destroy((LPCNetState *)st); }
void ref_state_reset(void *st) { lpcnet_reset((LPCNetState *)st); }
void ref_state_copy(void *dst, const void *src) { *(LPCNetState *)dst = *(const LPCNetState *)src; }   /* what lpcnet_plc.c:216-230 does */
void ref_synthesize_impl(void *st, const float *features, short *out, int N, int preload) { lpcnet_synthesize_impl((LPCNetState *)st, features, out, N, preload); }
void ref_run_frame_network(void *st, const float *features)
{
    LPCNetState *l = (LPCNetState *)st;
    run_frame_network(l, l->gru_a_condition, l->gru_b_condition, l->lpc, features);
}
void ref_synthesize_tail(void *st, short *out, int N, int preload) { lpcnet_synthesize_tail_impl((LPCNetState *)st, out, N, preload); }
void ref_frame_network_deferred(void *st, const float *features) { run_frame_network_deferred((LPCNetState *)st, features); }
void ref_frame_network_flush(void *st) { run_frame_network_flush((LPCNetState *)st); }
void ref_reset_signal(void *st) { lpcnet_reset_signal((LPCNetState *)st); }

/* ---- the decoder's state (LPCNetDecState, lpcnet_private.h:50-53) on an explicit handle.  It starts with its LPCNetState, so
 * the entry points above also take a decoder handle. ---- */
void *ref_dec_state_create(const unsigned char *blob, int len)
{
    LPCNetDecState *st = lpcnet_decoder_create();
    if (lpcnet_load_model((LPCNetState *)st, blob, len) != 0) { lpcnet_decoder_destroy(st); return NULL; }
    return st;
}
void ref_dec_state_destroy(void *st) { lpcnet_decoder_destroy((LPCNetDecState *)st); }
int ref_decode(void *st, const unsigned char *packet, short *pcm) { return lpcnet_decode((LPCNetDecState *)st, packet, pcm); }
/* what lpcnet_decoder_init does to a loaded state: lpcnet_reset, and the previous superframe's cepstrum cleared */
void ref_dec_reset(void *st)
{
    LPCNetDecState *d = (LPCNetDecState *)st;
    lpcnet_reset(&d->lpcnet_state);
    memset(d->vq_mem, 0, sizeof(d->vq_mem));
}
void ref_dec_state_copy(void *dst, const void *src) { *(LPCNetDecState *)dst = *(const LPCNetDecState *)src; }

/* ---- encoder / feature extraction (SURVEY 8f N2): the reference's own entry points on one stream with a fresh state ---- */
/* lpcnet_compute_single_frame_features (lpcnet_enc.c:919) per 160-sample frame: pcm [nframes*160] -> features [nframes][36] */
int ref_features_stream(const short *pcm, int nframes, float *features)
{
    int i;
    LPCNetEncState *st = lpcnet_encoder_create();
    for (i = 0; i < nframes; i++) lpcnet_compute_single_frame_features(st, pcm + (size_t)i * LPCNET_FRAME_SIZE, features + (size_t)i * NB_TOTAL_FEATURES);
    lpcnet_encoder_destroy(st);
    return 0;
}
int ref_features_stream_float(const float *pcm, int nframes, float *features)
{
    int i;
    LPCNetEncState *st = lpcnet_encoder_create();
    for (i = 0; i < nframes; i++) lpcnet_compute_single_frame_features_float(st, pcm + (size_t)i * LPCNET_FRAME_SIZE, features + (size_t)i * NB_TOTAL_FEATURES);
    lpcnet_encoder_destroy(st);
    return 0;
}
/* lpcnet_encode (lpcnet_enc.c:882) per 640-sample packet: pcm [npackets*640] -> packets [npackets][8] */
int ref_encode_stream(const short *pcm, int npackets, unsigned char *packets)
{
    int i;
    LPCNetEncState *st = lpcnet_encoder_create();
    for (i = 0; i < npackets; i++) lpcnet_encode(st, pcm + (size_t)i * LPCNET_PACKET_SAMPLES, packets + (size_t)i * LPCNET_COMPRESSED_SIZE);
    lpcnet_encoder_destroy(st);
    return 0;
}
/* lpcnet_compute_features (lpcnet_enc.c:896): unquantised 4-frame analysis, pcm [npackets*640] -> features [npackets*4][36] */
int ref_features4_stream(const short *pcm, int npackets, float *features)
{
    int i;
    LPCNetEncState *st = lpcnet_encoder_create();
    for (i = 0; i < npackets; i++) lpcnet_compute_features(st, pcm + (size_t)i * LPCNET_PACKET_SAMPLES, (float (*)[NB_TOTAL_FEATURES])(features + (size_t)i * 4 * NB_TOTAL_FEATURES));
    lpcnet_encoder_destroy(st);
    return 0;
}
/* a mixed call sequence on ONE state: encode, then single-frame analysis (pcount stays where lpcnet_encode left it) */
int ref_encode_then_features(const short *pcm, int npackets, unsigned char *packets, int nframes, float *features)
{
    int i;
    LPCNetEncState *st = lpcnet_encoder_create();
    for (i = 0; i < npackets; i++) lpcnet_encode(st, pcm + (size_t)i * LPCNET_PACKET_SAMPLES, packets + (size_t)i * LPCNET_COMPRESSED_SIZE);
    pcm += (size_t)npackets * LPCNET_PACKET_SAMPLES;
    for (i = 0; i < nframes; i++) lpcnet_compute_single_frame_features(st, pcm + (size_t)i * LPCNET_FRAME_SIZE, features + (size_t)i * NB_TOTAL_FEATURES);
    lpcnet_encoder_destroy(st);
    return 0;
}
extern const float half_window[];
extern const float dct_table[];
void ref_enc_tables(float *hw /*[160]*/, float *dct /*[324]*/) { memcpy(hw, half_window, sizeof(float) * OVERLAP_SIZE); memcpy(dct, dct_table, sizeof(float) * NB_BANDS * NB_BANDS); }

/* ---- many streams on a pool of host threads (golden generation at BASELINE sizes; work queue over streams) ---- */
typedef struct {
    const unsigned char *blob; int len; const float *features; int stride; int nframes; short *pcm;
    const unsigned char *packets; int npackets; int n_streams; volatile int *next; int rc;
} pool_t;

static void *pool_worker(void *arg)
{
    pool_t *p = (pool_t *)arg;
    for (;;) {
        int s = __sync_fetch_and_add(p->next, 1);
        if (s >= p->n_streams) break;
        if (p->packets) {
            if (ref_decode_stream(p->blob, p->len, p->packets + (size_t)s * p->npackets * LPCNET_COMPRESSED_SIZE, p->npackets,
                                  p->pcm + (size_t)s * p->npackets * LPCNET_PACKET_SAMPLES)) p->rc = -1;
        } else {
            if (ref_synth_stream(p->blob, p->len, p->features + (size_t)s * p->nframes * p->stride, p->stride, p->nframes,
                                 p->pcm + (size_t)s * p->nframes * LPCNET_FRAME_SIZE)) p->rc = -1;
        }
    }
    return NULL;
}

static int run_pool(pool_t *proto, int nthreads)
{
    pthread_t *th = malloc(sizeof(*th) * nthreads);
    pool_t *ps = malloc(sizeof(*ps) * nthreads);
    volatile int next = 0;
    int i, rc = 0;
    for (i = 0; i < nthreads; i++) { ps[i] = *proto; ps[i].next = &next; ps[i].rc = 0; pthread_create(&th[i], NULL, pool_worker, &ps[i]); }
    for (i = 0; i < nthreads; i++) { pthread_join(th[i], NULL); rc |= ps[i].rc; }
    free(th); free(ps);
    return rc;
}

/* features [n_streams][nframes][stride] -> pcm [n_streams][nframes*160], every stream from a fresh lpcnet_create() */
int ref_synth_batch(const unsigned char *blob, int len, const float *features, int stride, int nframes, int n_streams,
                    int nthreads, short *pcm)
{
    pool_t p; memset(&p, 0, sizeof(p));
    p.blob = blob; p.len = len; p.features = features; p.stride = stride; p.nframes = nframes; p.pcm = pcm; p.n_streams = n_streams;
    return run_pool(&p, nthreads);
}

/* packets [n_streams][npackets][8] -> pcm [n_streams][npackets*640] */
int ref_decode_batch(const unsigned char *blob, int len, const unsigned char *packets, int npackets, int n_streams,
                     int nthreads, short *pcm)
{
    pool_t p; memset(&p, 0, sizeof(p));
    p.blob = blob; p.len = len; p.packets = packets; p.npackets = npackets; p.pcm = pcm; p.n_streams = n_streams;
    return run_pool(&p, nthreads);
}

/* ---- CPU baseline timing (BASELINE.md 3): `nthreads` independent streams, one per host thread.  State creation and
 * model loading happen BEFORE the clock starts (all threads meet at a barrier); the timed region is the
 * lpcnet_synthesize / lpcnet_decode calls only.  Returns wall seconds from the barrier to the last thread's finish. ---- */
typedef struct {
    const unsigned char *blob; int len; const float *features; int stride; int nframes; short *pcm;
    const unsigned char *packets; pthread_barrier_t *bar; struct timespec t0, t1; int rc;
} tjob_t;

static void *timed_worker(void *arg)
{
    tjob_t *j = (tjob_t *)arg;
    int i;
    if (j->packets) {
        LPCNetDecState *st = lpcnet_decoder_create();
        j->rc = lpcnet_load_model((LPCNetState *)st, j->blob, j->len);
        pthread_barrier_wait(j->bar);
        clock_gettime(CLOCK_MONOTONIC, &j->t0);
        if (!j->rc) for (i = 0; i < j->nframes; i++)
            lpcnet_decode(st, j->packets + (size_t)i * LPCNET_COMPRESSED_SIZE, j->pcm + (size_t)i * LPCNET_PACKET_SAMPLES);
        clock_gettime(CLOCK_MONOTONIC, &j->t1);
        lpcnet_decoder_destroy(st);
    } else {
        LPCNetState *st = lpcnet_create();
        j->rc = lpcnet_load_model(st, j->blob, j->len);
        pthread_barrier_wait(j->bar);
        clock_gettime(CLOCK_MONOTONIC, &j->t0);
        if (!j->rc) for (i = 0; i < j->nframes; i++)
            lpcnet_synthesize(st, j->features + (size_t)i * j->stride, j->pcm + (size_t)i * LPCNET_FRAME_SIZE, LPCNET_FRAME_SIZE);
        clock_gettime(CLOCK_MONOTONIC, &j->t1);
        lpcnet_destroy(st);
    }
    return NULL;
}

/* features: [nthreads][nframes][stride] (or packets: [nthreads][nframes][8] when `packets` != NULL, nframes = packets per
 * stream); pcm: [nthreads][nframes*160] (or *640) */
double ref_time_streams(const unsigned char *blob, int len, const float *features, int stride, const unsigned char *packets,
                        int nframes, int nthreads, short *pcm)
{
    pthread_t *th = malloc(sizeof(*th) * nthreads);
    tjob_t *jobs = malloc(sizeof(*jobs) * nthreads);
    pthread_barrier_t bar;
    double first = 0, last = 0;
    int i;
    pthread_barrier_init(&bar, NULL, nthreads);
    for (i = 0; i < nthreads; i++) {
        memset(&jobs[i], 0, sizeof(jobs[i]));
        jobs[i].blob = blob; jobs[i].len = len; jobs[i].stride = stride; jobs[i].nframes = nframes; jobs[i].bar = &bar;
        if (packets) { jobs[i].packets = packets + (size_t)i * nframes * LPCNET_COMPRESSED_SIZE; jobs[i].pcm = pcm + (size_t)i * nframes * LPCNET_PACKET_SAMPLES; }
        else { jobs[i].features = features + (size_t)i * nframes * stride; jobs[i].pcm = pcm + (size_t)i * nframes * LPCNET_FRAME_SIZE; }
        pthread_create(&th[i], NULL, timed_worker, &jobs[i]);
    }
    for (i = 0; i < nthreads; i++) pthread_join(th[i], NULL);
    for (i = 0; i < nthreads; i++) {
        double a = jobs[i].t0.tv_sec + 1e-9 * jobs[i].t0.tv_nsec, b = jobs[i].t1.tv_sec + 1e-9 * jobs[i].t1.tv_nsec;
        if (i == 0 || a < first) first = a;
        if (i == 0 || b > last) last = b;
        if (jobs[i].rc) { last = first - 1; break; }
    }
    pthread_barrier_destroy(&bar);
    free(th); free(jobs);
    return last - first;     /* negative on error */
}
