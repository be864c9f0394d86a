// batch_api.cu — C-ABI of include/lpcnet_b200.h: batches of independent streams stepped in lockstep.
//
// Per call: [H2D features] -> (per chunk of <= CHUNK frames) frame network + LPC kernels -> persistent per-sample
// kernel -> [D2H PCM].  The per-stream state mirrors the resettable part of struct LPCNetState
// (reference src/lpcnet_private.h:28-48) in structure-of-arrays form (stream index fastest) so that lane==stream
// accesses coalesce.  Streams have their own lifecycle: each carries its own frame counter (silent warm-up frames after
// a reset, lpcnet.c:239-243), can be reset / exported / imported individually, and the whole batch can be snapshotted
// and rolled back on the device (what the reference's PLC does by copying LPCNetState by value, lpcnet_plc.c:216-230).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "engine.h"
#include "devmath.cuh"
#include "../../include/lpcnet_b200.h"

namespace lpcnet_b200 { const char *get_error(); }
using namespace lpcnet_b200;

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_error("%s failed: %s", #call, cudaGetErrorString(e_)); return -1; } } while (0)

static const int CHUNK = FRAME_CHUNK;   // frames of conditioning buffered per sample-kernel launch
static const int DEFER_MAX = 4;     // MAX_FEATURE_BUFFER_SIZE (lpcnet_private.h:26): conv1.kernel_size + conv2.kernel_size - 2
// One more conditioning frame past the chunk slots: the frame a tail reads once a flush, a reset or a restore has put it there.
// It plays the part of the reference's gru_a_condition / gru_b_condition / lpc, which a flush does not touch (lpcnet.c:134-144).
// Its LPC lives in lpc_raw entry CHUNK + 2, past the entries 0..CHUNK+1 a chunk writes.
static const int TAIL_SLOT = CHUNK;

// the sample-rate part of the per-stream state (resettable part of struct LPCNetState), structure of arrays
struct SampleState { float *hA, *hB, *last_sig, *deemph; int *last_exc; uint32_t *rng; };
// One frame of conditioning as the per-sample kernel reads it: condA (int8 [3 gates][n][na + 8], float [n][3*na]), condB [n][3*NB],
// raw LPC [n][16]
struct CondFrame { float *A, *B, *L; };
// device buffers of a copy of the per-stream state (a batch's shadow copy, a snapshot), for the parts it was allocated for
struct StateCopy { SampleState ss; FrameState fs; CondFrame tail; };

// Chunks of PCM forwarded to PcmTargets (a batch's sink, the gather buffer of a multi-GPU group) on a copy stream that overlaps
// the next chunk's kernels; the stream is made on first use
struct PcmForwarder {
    cudaStream_t stream; cudaEvent_t ev, done;     // ev: the copy stream's hand-over event
    int open()
    {
        if (stream) return 0;
        CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
        return 0;
    }
    // chunk [c0, c0+nf) of the n PCM rows at d_pcm is complete on `st`: its block goes to t
    int forward_to_sink(const PcmTarget &t, int n, const short *d_pcm, long long pcm_stride, int c0, int nf, int spf, cudaStream_t st)
    {
        CK(cudaEventRecord(ev, st));
        CK(cudaStreamWaitEvent(stream, ev, 0));
        short *dst = t.dst + t.row0 * t.pitch + (size_t)c0 * spf;
        if (c0 == 0 && (long long)nf * spf == pcm_stride && t.pitch == pcm_stride)      // whole rows, same pitch: one contiguous block (one DMA descriptor
            CK(cudaMemcpyAsync(dst, d_pcm, (size_t)n * pcm_stride * sizeof(short), cudaMemcpyDefault, stream));   // instead of n row copies)
        else
            CK(cudaMemcpy2DAsync(dst, t.pitch * sizeof(short), d_pcm + (size_t)c0 * spf, pcm_stride * sizeof(short), (size_t)nf * spf * sizeof(short), n,
                                 cudaMemcpyDefault, stream));       // (the target may live on another device: UVA infers the route)
        return 0;
    }
    int join(cudaStream_t st)        // the call's stream also waits for the forwarded copies: "call complete" includes "PCM at the target"
    {
        CK(cudaEventRecord(done, stream));
        CK(cudaStreamWaitEvent(st, done, 0));
        return 0;
    }
    void destroy()
    {
        if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }
        if (ev) cudaEventDestroy(ev);
        if (done) cudaEventDestroy(done);
    }
};

struct LPCNetB200Batch {
    int device, n;
    DeviceModel model;
    FrameState fs;
    SampleState ss;
    StateCopy shadow;                             // scratch copy for calls in which only SOME streams advance: the sample-rate part for frames
                                                  // some streams sit out in their silent warm-up, the 100 Hz part for flushes some have no frame for
    int *d_mask;                                  // [DEFER_MAX][n] per frame of such a call: 1 = the stream sits the frame out
    std::vector<int> fc;                          // host mirror of fs.frame_count
    // work buffers: CHUNK chunk slots + TAIL_SLOT
    float *condA, *condB, *lpc_raw;
    int cond_last;                                // slot of the conditioning a tail reads (a chunk position or TAIL_SLOT); -1 = none since an import
    float *d_features; size_t d_features_cap;     // staging for host-pointer calls / decoder output
    short *d_pcm; size_t d_pcm_cap;
    uint8_t *d_packets; size_t d_packets_cap;
    float *d_state; size_t d_state_cap;           // staging for export/import of one stream's state and for copies between batches
    // run_frame_network_deferred queue: [DEFER_MAX][n][20] on the host, deferred_fill frames long.  Stream s has queued the LAST
    // dfill[s] <= deferred_fill of them (a reset or an import empties one stream's queue, lpcnet.c:174-182).
    std::vector<float> deferred; int deferred_fill; std::vector<int> dfill;
    cudaStream_t stream;
    // Ordering of the engine state across CUDA streams: every call that enqueues work records `order_ev` on the stream it
    // used; the next call makes ITS stream wait for that event first (and host-side readers synchronise on it).  A caller
    // may therefore pass a different cuda_stream to every `_device` call, or mix them with the host-pointer calls.
    cudaEvent_t order_ev; cudaStream_t last_stream; bool has_order;
    int env_spc;                                  // LPCNET_B200_STREAMS_PER_CTA (0: automatic)
    bool env_exact_cvt, env_float_lane_stream, env_two_halves;    // LPCNET_B200_EXACT_CVT / _FLOAT_LANE_STREAM / _TWO_HALVES, read once at create time (tests)
    cudaEvent_t ev0, ev1;                         // user timer (lpcnet_b200_batch_timer_*)
    std::vector<cudaEvent_t> kev;                 // event pairs around every per-sample kernel launch of the last call
    int kev_used;
    int last_launches;
    // PCM sink (multi-GPU gather): after every chunk the chunk's PCM block is also forwarded to the sink (a buffer of another
    // device / another process opened through CUDA IPC)
    PcmTarget sink; PcmForwarder fwd;
};

int lpcnet_b200::grow_buffer(void **p, size_t *cap, size_t bytes)
{
    if (*cap >= bytes) return 0;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    CK(cudaMalloc(p, bytes));
    *cap = bytes;
    return 0;
}
static int order_sync(LPCNetB200Batch *b);
// grow a staging buffer; work on any stream may still be using the old one, so wait for it before freeing
static int ensure(LPCNetB200Batch *b, void **p, size_t *cap, size_t bytes)
{
    if (*cap >= bytes) return 0;
    return order_sync(b) || grow_buffer(p, cap, bytes) ? -1 : 0;
}

// stream hand-over (see LPCNetB200Batch::order_ev)
static int order_enter(LPCNetB200Batch *b, cudaStream_t st)
{
    if (b->has_order && b->last_stream != st) CK(cudaStreamWaitEvent(st, b->order_ev, 0));
    return 0;
}
static int order_leave(LPCNetB200Batch *b, cudaStream_t st)
{
    CK(cudaEventRecord(b->order_ev, st));
    b->last_stream = st; b->has_order = true;
    return 0;
}
static int order_sync(LPCNetB200Batch *b)       // host-side readers / writers of the state: wait for whatever ran last
{
    if (b->has_order) CK(cudaEventSynchronize(b->order_ev));
    return 0;
}

// The RCPPS look-up of the per-sample kernel forms its table address as `table | index` (devmath.cuh), which needs the
// table 8 KB-aligned in the SHARED WINDOW; the image offsets assume dynamic shared memory starts at SMEM_RESERVED.
// Probed once per device at create time so that a driver with a different reservation fails here with a message,
// not with a trap inside the kernel.
__global__ void smem_base_probe_kernel(uint32_t *out)
{
    extern __shared__ __align__(128) uint8_t probe_smem[];
    *out = (uint32_t)__cvta_generic_to_shared(probe_smem);
}
static int probe_smem_base(uint32_t *base)
{
    uint32_t *d = nullptr;
    CK(cudaMalloc(&d, 4));
    CK(cudaFuncSetAttribute(smem_base_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    smem_base_probe_kernel<<<1, 32, 227 * 1024>>>(d);
    cudaError_t e = cudaMemcpy(base, d, 4, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) { set_error("shared-memory probe failed: %s", cudaGetErrorString(e)); return -1; }
    return 0;
}

// The launch plan of a batch (one member) and of a group.  Live streams per CTA: a job smaller than 32 x SM count is spread over
// all SMs (fewer live slots per CTA) instead of filling a few SMs completely: the time of a CTA-step barely depends on how many of
// its slots are live.  One streams-per-CTA value for the whole launch: the smallest that puts every member on at most `sms` CTAs in
// total, member k on ceil(n_k / spc) CTAs of its own; 32 when none does (LPCNET_B200_STREAMS_PER_CTA overrides it, clamped to 32).
static int group_plan(const int *n, int count, int sms, int override_spc, int *ctas)
{
    auto total = [&](int spc) { int c = 0; for (int k = 0; k < count; k++) c += (n[k] + spc - 1) / spc; return c; };
    int spc = STREAMS_PER_CTA;
    if (override_spc > 0) spc = std::min(override_spc, STREAMS_PER_CTA);
    else for (int s = 1; s <= STREAMS_PER_CTA; s++) if (total(s) <= sms) { spc = s; break; }
    *ctas = total(spc);
    return spc;
}
// The float flavour takes spc from group_plan and then its kernel: at spc <= FN_S, unless LPCNET_B200_FLOAT_LANE_STREAM is set,
// the neuron-per-lane kernel, whose CTAs lay out S = 1, 2 or FN_S streams (spc 3 -> 4); otherwise the lane == stream kernel with
// spc.  Returns the streams a CTA lays out (member k takes ceil(n_k / slots) CTAs); *neuron: the neuron-per-lane kernel.
static int float_slots(int spc, bool lane_stream, bool *neuron)
{
    *neuron = spc <= FN_S && !lane_stream;
    return !*neuron ? spc : spc <= 1 ? 1 : spc == 2 ? 2 : FN_S;
}
int lpcnet_b200::sample_kernel_smem_ok(uint32_t bytes) { return bytes <= 227u * 1024u; }

#ifdef LPCNET_TRACE
static long long *g_trace = nullptr;
extern "C" __attribute__((visibility("default"))) int lpcnet_b200_debug_read_trace(long long *out)
{
    if (!g_trace) return -1;
    cudaDeviceSynchronize();
    return cudaMemcpy(out, g_trace, (8 * 32 + 8 * 32 * 16) * 8, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;   // + [8 samples][32 warps][16 events] per-warp stamps
}
#endif

// kiss99_srand(&rng, "LPCNet", 6): reference src/kiss99.c:32-57 called from lpcnet_reset (src/lpcnet.c:176-181).
static void kiss99_seed(uint32_t st[4])
{
    const unsigned char *d = (const unsigned char *)"LPCNet"; const int nd = 6;
    uint32_t z = 362436069u, w = 521288629u, jsr = 123456789u, jcong = 380116160u;
    int i;
    for (i = 3; i < nd; i += 4) {
        z ^= d[i - 3]; w ^= d[i - 2]; jsr ^= d[i - 1]; jcong ^= d[i];
        uint32_t znew = 36969u * (z & 0xFFFF) + (z >> 16), wnew = 18000u * (w & 0xFFFF) + (w >> 16);
        uint32_t shr3 = jsr ^ (jsr << 13); shr3 ^= shr3 >> 17; shr3 ^= shr3 << 5;
        z = znew; w = wnew; jsr = shr3; jcong = 69069u * jcong + 1234567u;
    }
    if (i - 3 < nd) z ^= d[i - 3];
    if (i - 2 < nd) w ^= d[i - 2];
    if (i - 1 < nd) jsr ^= d[i - 1];
    if (z == 0 || z == 0x9068FFFF) z++;
    if (w == 0 || w == 0x464FFFFF) w++;
    if (jsr == 0) jsr++;
    st[0] = z; st[1] = w; st[2] = jsr; st[3] = jcong;
}

// ------------------------------------------------------------------------------------------------------------------
// The per-stream state as one field table: allocation, copies, resets, roll-backs and the by-value record all follow it.
// `part` says which operations touch a field: reset_signal clears SIGNAL only (the RNG belongs to the sample rate, but
// lpcnet_reset_signal keeps it, lpcnet.c:226-233); FRAME is the 100 Hz state; TAIL is the stream's row of the conditioning
// frame a tail reads (the reference's gru_a_condition / gru_b_condition / lpc).
enum : unsigned { SIGNAL = 1, RNG = 2, FRAME = 4, TAIL = 8, STATE = SIGNAL | RNG | FRAME, ALL = STATE | TAIL };
// Word i of stream s: base[(i / width) * n * pitch + s * pitch + i % width].  `slot` is the owner's pointer (allocation, freeing).
struct Field { float *base; int planes, width, pitch; unsigned part; void **slot; };
// record order: the exported words (oracle_export_state), then the tail part a copy between batches adds
enum { F_HA, F_HB, F_LAST_SIG, F_DEEMPH, F_CONV1, F_CONV2, F_LPC_CARRY, F_VQ_MEM, F_LAST_EXC, F_FRAME_COUNT, F_RNG, F_COND_A, F_COND_B, F_COND_L, NFIELDS };
struct Fields { Field f[NFIELDS]; int n; };

static Fields state_fields(SampleState &ss, FrameState &fs, CondFrame &tail, int n, int na, int a_float)
{
    auto field = [](auto *&p, int planes, int width, int pitch, unsigned part) { return Field{(float *)p, planes, width, pitch, part, (void **)&p}; };
    auto soa = [&](auto *&p, int count, unsigned part) { return field(p, count, 1, 1, part); };        // [count][n]
    auto row = [&](auto *&p, int count, unsigned part) { return field(p, 1, count, count, part); };    // [n][count]
    return Fields{{soa(ss.hA, na, SIGNAL), soa(ss.hB, NB, SIGNAL), soa(ss.last_sig, LPC_ORDER, SIGNAL), soa(ss.deemph, 1, SIGNAL),
                   row(fs.conv1_state, 2 * FRAME_IN, FRAME), row(fs.conv2_state, 2 * COND, FRAME), field(fs.lpc_carry, 2, LPC_ORDER, LPC_ORDER, FRAME),
                   row(fs.vq_mem, NB_BANDS, FRAME), soa(ss.last_exc, 1, SIGNAL), row(fs.frame_count, 1, FRAME), soa(ss.rng, 4, RNG),
                   a_float ? row(tail.A, 3 * na, TAIL) : field(tail.A, 3, na, na + 8, TAIL), row(tail.B, 3 * NB, TAIL), row(tail.L, LPC_ORDER, TAIL)}, n};
}
// words of the record in front of field `end` (NFIELDS: the whole record)
static int record_words(const Fields &t, int end)
{
    int w = 0;
    for (int j = 0; j < end; j++) w += t.f[j].planes * t.f[j].width;
    return w;
}
static int record_words(int na, int end) { SampleState ss{}; FrameState fs{}; CondFrame tail{}; return record_words(state_fields(ss, fs, tail, 0, na, 0), end); }
// words of one stream's exported state, and the words a copy between batches adds behind them
static int state_words(int na) { return record_words(na, F_COND_A); }
static int tail_words(int na) { return record_words(na, NFIELDS) - state_words(na); }

static size_t field_floats(const Field &f, size_t n) { return (size_t)f.planes * n * f.pitch; }
static bool alloc_state(const Fields &t, unsigned parts)
{
    for (const Field &f : t.f) if ((f.part & parts) && !*f.slot && cudaMalloc(f.slot, sizeof(float) * field_floats(f, t.n)) != cudaSuccess) return false;
    return true;
}
static void free_state(const Fields &t)
{
    for (const Field &f : t.f) if (f.slot && *f.slot) { cudaFree(*f.slot); *f.slot = nullptr; }
}
static int copy_state(const Fields &dst, const Fields &src, unsigned parts, cudaStream_t st)
{
    for (int j = 0; j < NFIELDS; j++)
        if (src.f[j].part & parts)
            CK(cudaMemcpyAsync(dst.f[j].base, src.f[j].base, sizeof(float) * field_floats(src.f[j], src.n), cudaMemcpyDeviceToDevice, st));
    return 0;
}

// per-stream state kernels (rare paths: resets, export / import, copies between batches, mixed silent segments, partial flushes)
__device__ inline size_t field_word(const Field &f, size_t n, size_t s, int i) { return (size_t)(i / f.width) * n * f.pitch + s * f.pitch + i % f.width; }
// one block per record k of buf (`words` apart; 0: every stream reads the same record): stream rows[k] (rows == NULL: stream s0 + k).
// The fields of `parts` move, each at its place in the record.  UNPACK: record -> stream.
template <bool UNPACK>
__global__ void records_kernel(Fields t, const int *rows, int s0, float *buf, int words, unsigned parts)
{
    const int k = blockIdx.x;
    const size_t s = rows ? rows[k] : s0 + k;
    float *rec = buf + (size_t)k * words;
    for (int j = 0, o = 0; j < NFIELDS; o += t.f[j].planes * t.f[j].width, j++) {
        const Field &f = t.f[j];
        if (!(f.part & parts)) continue;
        for (int i = threadIdx.x; i < f.planes * f.width; i += blockDim.x) {
            float *p = f.base + field_word(f, t.n, s, i);
            if (UNPACK) *p = rec[o + i]; else rec[o + i] = *p;
        }
    }
}
// dst <- src, the fields of `parts`, for the streams s with mask[s] set; their `spf` samples at pcm + s * pcm_stride become zeros (pcm != NULL)
__global__ void restore_masked_kernel(Fields dst, Fields src, const int *mask, unsigned parts, short *pcm, long long pcm_stride, int spf)
{
    const size_t s = blockIdx.x;
    if (!mask[s]) return;
    for (int j = 0; j < NFIELDS; j++) {
        const Field &f = dst.f[j];
        if (!(f.part & parts)) continue;
        for (int i = threadIdx.x; i < f.planes * f.width; i += blockDim.x) {
            const size_t w = field_word(f, dst.n, s, i);
            f.base[w] = src.f[j].base[w];
        }
    }
    if (pcm) for (int i = threadIdx.x; i < spf; i += blockDim.x) pcm[s * pcm_stride + i] = 0;
}

// the conditioning the per-sample kernel reads for the frame in slot `pos`; frame f of a chunk reads lpc_raw entry f + 2 - d
// (frame_kernels.cu), TAIL_SLOT its own entry
static CondFrame frame_at(const LPCNetB200Batch *b, int pos)
{
    const size_t n = b->n;
    const int d = b->model.cfg.end2end ? 0 : b->model.cfg.features_delay;
    const size_t e = pos == TAIL_SLOT ? CHUNK + 2 : pos + 2 - d;
    return CondFrame{b->condA + pos * condA_frame_floats(b->model.is_float != 0, n, b->model.na), b->condB + pos * n * 3 * NB, b->lpc_raw + e * n * LPC_ORDER};
}
// the batch's state, with the frame in slot `pos` as its tail (pos < 0: none).  The tail is not the batch's own allocation: no slots.
static Fields batch_fields(LPCNetB200Batch *b, int pos)
{
    CondFrame tail = pos >= 0 ? frame_at(b, pos) : CondFrame{};
    Fields t = state_fields(b->ss, b->fs, tail, b->n, b->model.na, b->model.is_float);
    for (int j = F_COND_A; j < NFIELDS; j++) t.f[j].slot = nullptr;
    return t;
}
static Fields shadow_fields(LPCNetB200Batch *b) { return state_fields(b->shadow.ss, b->shadow.fs, b->shadow.tail, b->n, b->model.na, b->model.is_float); }
// move the frame a tail reads into TAIL_SLOT, out of the chunk slots the next frame-network run overwrites
static int park_tail(LPCNetB200Batch *b, cudaStream_t st)
{
    if (b->cond_last < 0 || b->cond_last == TAIL_SLOT) return 0;
    if (copy_state(batch_fields(b, TAIL_SLOT), batch_fields(b, b->cond_last), TAIL, st)) return -1;
    b->cond_last = TAIL_SLOT;
    return 0;
}

extern "C" {

int lpcnet_b200_version(void) { return 200; }
const char *lpcnet_b200_last_error(void) { return get_error(); }

int lpcnet_b200_device_count(void)
{
    int c = 0;
    if (cudaGetDeviceCount(&c) != cudaSuccess) { cudaGetLastError(); return 0; }
    return c;
}

// lpcnet_reset (lpcnet.c:174-182) for the listed streams (ids == NULL: all n streams); signal_only = lpcnet_reset_signal (lpcnet.c:226-233).
// A fresh record is unpacked into every listed stream: zeros, last_exc = lin2ulaw(0.f) = 128 (lpcnet.c:180), the kiss99 seed of the RNG.
static int reset_impl(LPCNetB200Batch *b, const int *ids, int count, int signal_only)
{
    CK(cudaSetDevice(b->device));
    if (ids) for (int k = 0; k < count; k++) if (ids[k] < 0 || ids[k] >= b->n) { set_error("reset_streams: stream %d out of range", ids[k]); return -1; }
    // a full reset of every stream leaves the zeroed TAIL_SLOT as what a tail reads; a per-stream one zeroes the streams' part of
    // the current tail frame (as the reference clears gru_a_condition, gru_b_condition and lpc; none since an import: tails stay
    // refused until the next frame-network run)
    if (!signal_only && !ids) b->cond_last = TAIL_SLOT;
    const Fields t = batch_fields(b, b->cond_last);
    const int words = record_words(t, NFIELDS), last_exc = 128;
    uint32_t seed[4];
    kiss99_seed(seed);
    std::vector<float> rec(words, 0.f);
    memcpy(&rec[record_words(t, F_LAST_EXC)], &last_exc, sizeof(last_exc));
    memcpy(&rec[record_words(t, F_RNG)], seed, sizeof(seed));
    // staging: the record, then the stream ids
    if (ensure(b, (void **)&b->d_state, &b->d_state_cap, sizeof(float) * words + (ids ? sizeof(int) * count : 0))) return -1;
    int *d_ids = ids ? reinterpret_cast<int *>(b->d_state + words) : nullptr;
    if (order_enter(b, b->stream)) return -1;
    CK(cudaMemcpyAsync(b->d_state, rec.data(), sizeof(float) * words, cudaMemcpyHostToDevice, b->stream));
    if (ids) CK(cudaMemcpyAsync(d_ids, ids, sizeof(int) * count, cudaMemcpyHostToDevice, b->stream));
    records_kernel<true><<<count, 128, 0, b->stream>>>(t, d_ids, 0, b->d_state, 0, signal_only ? SIGNAL : b->cond_last >= 0 ? ALL : STATE);
    if (order_leave(b, b->stream)) return -1;
    CK(cudaStreamSynchronize(b->stream));
    if (!signal_only) {
        if (ids) for (int k = 0; k < count; k++) { b->fc[ids[k]] = 0; b->dfill[ids[k]] = 0; }
        else { std::fill(b->fc.begin(), b->fc.end(), 0); std::fill(b->dfill.begin(), b->dfill.end(), 0); b->deferred_fill = 0; }
    }
    return 0;
}

int lpcnet_b200_batch_reset(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return -1; }
    return reset_impl(b, nullptr, b->n, 0);
}
int lpcnet_b200_batch_reset_streams(LPCNetB200Batch *b, const int *streams, int count)
{
    if (!b || !streams || count < 0) { set_error("reset_streams: bad arguments"); return -1; }
    return count ? reset_impl(b, streams, count, 0) : 0;
}
int lpcnet_b200_batch_reset_signal(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return -1; }
    return reset_impl(b, nullptr, b->n, 1);
}

LPCNetB200Batch *lpcnet_b200_batch_create_ex(int n_streams, const unsigned char *blob, int blob_len, const LPCNetB200Config *cfg, int device)
{
    if (n_streams <= 0) { set_error("n_streams must be positive"); return nullptr; }
    int cnt = lpcnet_b200_device_count();
    if (cnt <= 0) { set_error("no CUDA device available (this engine has no CPU fallback)"); return nullptr; }
    if (device < 0 || device >= cnt) { set_error("device %d out of range (%d devices)", device, cnt); return nullptr; }
    if (cudaSetDevice(device) != cudaSuccess) { set_error("cudaSetDevice(%d) failed", device); return nullptr; }
    LPCNetB200Batch *b = new LPCNetB200Batch();
    b->device = device; b->n = n_streams; b->cond_last = -1;
    b->fc.assign(n_streams, 0);
    b->dfill.assign(n_streams, 0);
    ModelConfig mc{-1.f, -1, -1};
    if (cfg) { mc.lpc_gamma = cfg->lpc_gamma; mc.features_delay = cfg->features_delay; mc.end2end = cfg->end2end; }
    if (model_load(&b->model, blob, blob_len, &mc) != 0) { delete b; return nullptr; }
    const size_t n = n_streams;
    const int na = b->model.na;
    // the exported record is oracle_export_state's (lpcnet_b200_batch_state_size); a copy between batches adds the tail part
    if (state_words(na) != na + 513 || tail_words(na) != 3 * na + 64) {
        set_error("state record of %d words + %d tail words, expected %d + %d", state_words(na), tail_words(na), na + 513, 3 * na + 64);
        lpcnet_b200_batch_destroy(b); return nullptr;
    }
    bool ok = alloc_state(batch_fields(b, -1), STATE);
    auto al = [&](void **p, size_t bytes) { if (ok && cudaMalloc(p, bytes) != cudaSuccess) ok = false; };
    al((void **)&b->fs.work, sizeof(float) * frame_work_floats(n));
    al((void **)&b->condA, sizeof(float) * (size_t)(CHUNK + 1) * condA_frame_floats(b->model.is_float != 0, n, na)); al((void **)&b->condB, sizeof(float) * (size_t)(CHUNK + 1) * n * 3 * NB);
    al((void **)&b->lpc_raw, sizeof(float) * (size_t)(CHUNK + 3) * n * LPC_ORDER);
    if (ok && cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) ok = false;
    if (ok && (cudaStreamCreateWithFlags(&b->fs.side, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&b->fs.ev_fork, cudaEventDisableTiming) != cudaSuccess ||
               cudaEventCreateWithFlags(&b->fs.ev_join, cudaEventDisableTiming) != cudaSuccess)) ok = false;
    if (ok && (cudaEventCreate(&b->ev0) != cudaSuccess || cudaEventCreate(&b->ev1) != cudaSuccess)) ok = false;
    if (ok && cudaEventCreateWithFlags(&b->order_ev, cudaEventDisableTiming) != cudaSuccess) ok = false;
    { const char *e = getenv("LPCNET_B200_STREAMS_PER_CTA"); b->env_spc = e ? atoi(e) : 0; }
    b->env_exact_cvt = getenv("LPCNET_B200_EXACT_CVT") != nullptr;
    b->env_float_lane_stream = getenv("LPCNET_B200_FLOAT_LANE_STREAM") != nullptr;
    b->env_two_halves = getenv("LPCNET_B200_TWO_HALVES") != nullptr;
    if (!ok) { set_error("device allocation failed: %s", cudaGetErrorString(cudaGetLastError())); lpcnet_b200_batch_destroy(b); return nullptr; }
    if (!b->model.is_float) {
        uint32_t base = 0;
        const Geom G = make_geom(na);
        if (probe_smem_base(&base)) { lpcnet_b200_batch_destroy(b); return nullptr; }
        if ((base + G.sm_image + G.im_rcp) % 8192u != 0) {
            set_error("dynamic shared memory starts at window offset %u on this driver, the image layout assumes %u (engine.h SMEM_RESERVED)", base, SMEM_RESERVED);
            lpcnet_b200_batch_destroy(b); return nullptr;
        }
    }
    if (lpcnet_b200_batch_reset(b) != 0) { lpcnet_b200_batch_destroy(b); return nullptr; }
    return b;
}

LPCNetB200Batch *lpcnet_b200_batch_create(int n_streams, const unsigned char *blob, int blob_len, float lpc_gamma, int device)
{
    LPCNetB200Config c = {lpc_gamma, -1, -1};       // FEATURES_DELAY / END2END: the blob's metadata record if it has one, else 2 / 0
    return lpcnet_b200_batch_create_ex(n_streams, blob, blob_len, &c, device);
}

void lpcnet_b200_batch_destroy(LPCNetB200Batch *b)
{
    if (!b) return;
    cudaSetDevice(b->device);
    if (b->order_ev && b->has_order) cudaEventSynchronize(b->order_ev);     // the last call's work may sit on a caller stream
    if (b->stream) cudaStreamSynchronize(b->stream);
    if (b->fs.side) { cudaStreamSynchronize(b->fs.side); cudaStreamDestroy(b->fs.side); }
    if (b->fs.ev_fork) cudaEventDestroy(b->fs.ev_fork);
    if (b->fs.ev_join) cudaEventDestroy(b->fs.ev_join);
    b->fwd.destroy();
    free_state(batch_fields(b, -1)); free_state(shadow_fields(b));
    void *ptrs[] = {b->fs.work, b->condA, b->condB, b->lpc_raw, b->d_features, b->d_pcm, b->d_packets, b->d_state, b->d_mask};
    for (void *p : ptrs) if (p) cudaFree(p);
    for (cudaEvent_t e : b->kev) cudaEventDestroy(e);
    model_free(&b->model);
    if (b->ev0) cudaEventDestroy(b->ev0);
    if (b->ev1) cudaEventDestroy(b->ev1);
    if (b->order_ev) cudaEventDestroy(b->order_ev);
    if (b->stream) cudaStreamDestroy(b->stream);
    delete b;
}

int lpcnet_b200_batch_streams(const LPCNetB200Batch *b) { return b ? b->n : 0; }
int lpcnet_b200_batch_is_float(const LPCNetB200Batch *b) { return b ? b->model.is_float : -1; }
int lpcnet_b200_batch_model_info(const LPCNetB200Batch *b, int *gru_a_units, LPCNetB200Config *cfg)
{
    if (!b) { set_error("null batch"); return -1; }
    if (gru_a_units) *gru_a_units = b->model.na;
    if (cfg) { cfg->lpc_gamma = b->model.cfg.lpc_gamma; cfg->features_delay = b->model.cfg.features_delay; cfg->end2end = b->model.cfg.end2end; }
    return 0;
}

int lpcnet_b200_batch_set_codebooks(LPCNetB200Batch *b, const float *cb, size_t n_floats)
{
    if (!b) { set_error("null batch"); return -1; }
    const size_t want = 3 * 1024 * 17 + 4096 * 18;
    if (!cb || n_floats != want) { set_error("codebooks: expected %zu floats", want); return -1; }
    CK(cudaSetDevice(b->device));
    if (!b->model.codebooks) CK(cudaMalloc((void **)&b->model.codebooks, want * sizeof(float)));
    // ordered like any other call: a decode still queued on a caller stream reads the codebooks it was called with
    if (order_enter(b, b->stream)) return -1;
    CK(cudaMemcpyAsync(b->model.codebooks, cb, want * sizeof(float), cudaMemcpyHostToDevice, b->stream));
    if (order_leave(b, b->stream)) return -1;
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}

// the per-sample kernel's parameters for `nf` frames of batch b whose conditioning sits at chunk position `pos`, except the
// launch geometry and the rounding switch (spc, one_half, fast_cvt)
static SampleParams sample_params(const LPCNetB200Batch *b, int pos, int nf, int spf, short *pcm, long long pcm_stride)
{
    SampleParams p = {};
    p.L = b->model.L; p.image = b->model.image;
    p.emb_sig = b->model.emb_sig; p.emb_pred = b->model.emb_pred; p.emb_exc = b->model.emb_exc; p.fcw = b->model.fcw;
    const CondFrame c = frame_at(b, pos);
    p.condA = c.A; p.condB = c.B; p.lpc_raw = c.L;
    p.gamma_pow = b->model.gamma_pow;
    p.hA = b->ss.hA; p.hB = b->ss.hB; p.last_sig = b->ss.last_sig; p.deemph = b->ss.deemph; p.last_exc = b->ss.last_exc; p.rng = b->ss.rng;
    p.pcm = pcm;
    p.pcm_stream_stride = pcm_stride;
    p.n_streams = b->n; p.nframes = nf; p.spf = spf;
    return p;
}
// conversion-free rounding allowed for the batch's launches (env LPCNET_B200_EXACT_CVT: force the conversion-unit path, tests)
static bool batch_fast_cvt(const LPCNetB200Batch *b) { return b->model.fast_cvt && !b->env_exact_cvt; }

// an event pair around a per-sample launch, resolved lazily by lpcnet_b200_*_last_sample_kernel_ms (no sync here)
static int time_launch(std::vector<cudaEvent_t> &kev, int *used, cudaStream_t st)
{
    while ((int)kev.size() < *used + 1) { cudaEvent_t e; CK(cudaEventCreate(&e)); kev.push_back(e); }
    CK(cudaEventRecord(kev[*used], st));
    ++*used;
    return 0;
}
static float timed_ms(const std::vector<cudaEvent_t> &kev, int used)
{
    float total = 0.f;
    for (int i = 0; i + 1 < used; i += 2) {
        float ms = 0.f;
        if (cudaEventSynchronize(kev[i + 1]) != cudaSuccess) return -1.f;
        if (cudaEventElapsedTime(&ms, kev[i], kev[i + 1]) != cudaSuccess) return -1.f;
        total += ms;
    }
    return total;
}

// launch the per-sample kernel for `nf` frames whose conditioning sits at chunk position `pos`
static int launch_sample(LPCNetB200Batch *b, int pos, int nf, int spf, short *pcm, long long pcm_stride, int preload, cudaStream_t st, bool time_it)
{
    const int n = b->n, na = b->model.na;
    SampleParams p = sample_params(b, pos, nf, spf, pcm, pcm_stride);
    int ctas;
    bool small_float = false;       // small batch: the neuron-per-lane float kernel
    p.spc = group_plan(&n, 1, device_sms(b->device), b->env_spc, &ctas);
    if (b->model.is_float) float_slots(p.spc, b->env_float_lane_stream, &small_float);
    p.one_half = p.spc <= HALF && !b->env_two_halves;
    p.fast_cvt = (batch_fast_cvt(b) ? 1 : 0) | (preload << 8);
#ifdef LPCNET_TRACE
    { static long long *d_trace = nullptr; if (!d_trace) { CK(cudaMalloc(&d_trace, (8 * 32 + 8 * 32 * 16) * 8)); CK(cudaMemset(d_trace, 0, (8 * 32 + 8 * 32 * 16) * 8)); } p.trace = d_trace; g_trace = d_trace; }
#endif
    if (time_it && time_launch(b->kev, &b->kev_used, st)) return -1;
    if (small_float) { p.L = b->model.Ln; p.image = b->model.image_n; }
    cudaError_t e;
#define LPCNET_DISPATCH(ns) (small_float ? ns::launch_sample_kernel_f32n(p, st) : b->model.is_float ? ns::launch_sample_kernel_f32(p, st) : ns::launch_sample_kernel(p, st))
    switch (na) {
    case 128: e = LPCNET_DISPATCH(na128); break;
    case 256: e = LPCNET_DISPATCH(na256); break;
    default:  e = LPCNET_DISPATCH(na384); break;
    }
#undef LPCNET_DISPATCH
    if (e != cudaSuccess) { set_error("per-sample kernel launch failed: %s", cudaGetErrorString(e)); return -1; }
    if (time_it && time_launch(b->kev, &b->kev_used, st)) return -1;
    return 0;
}

// The sample loops of the frames at chunk positions [pos0, pos0 + nf): per stream, frames whose post-increment frame
// counter is <= FEATURES_DELAY are silent and do not advance the sample state (lpcnet.c:239-243).  b->fc = the streams'
// counters before frame pos0 (host mirror).  sample_prefix handles the frames that are silent for at least one stream (zeros,
// or one launch per frame with the still-silent streams put back) and returns in *live0 the first frame every stream runs;
// frames [*live0, nf) then take one launch.  Returns the number of engine kernels launched, < 0 on error.
static int sample_prefix(LPCNetB200Batch *b, int pos0, int nf, int spf, short *pcm, long long pcm_stride, int preload, cudaStream_t st, int *live0)
{
    const int n = b->n, delay = b->model.cfg.features_delay;
    int fc_min = 1 << 30, fc_max = 0;
    for (int v : b->fc) { fc_min = std::min(fc_min, v); fc_max = std::max(fc_max, v); }
    const int sil_all = std::min(nf, std::max(0, delay - fc_max));     // frames silent for EVERY stream
    const int sil_any = std::min(nf, std::max(0, delay - fc_min));     // frames silent for at least one stream
    int launches = 0;
    if (sil_all > 0) CK(cudaMemset2DAsync(pcm, pcm_stride * sizeof(short), 0, (size_t)sil_all * spf * sizeof(short), n, st));
    if (sil_any > sil_all) {
        // mixed segment (some streams were reset later than others): one launch per frame over all streams, then the streams
        // that are still silent get their sample-rate state back and zeros as output (lpcnet.c:239-243: RNN_CLEAR(output),
        // return — nothing advances)
        static_assert(MAX_FEATURES_DELAY <= DEFER_MAX, "silent frames of a segment fit the mask");
        if (!alloc_state(shadow_fields(b), SIGNAL | RNG)) { set_error("mixed silent segment: device allocation failed"); return -1; }
        const Fields cur = batch_fields(b, -1), old = shadow_fields(b);
        if (!b->d_mask) CK(cudaMalloc((void **)&b->d_mask, sizeof(int) * DEFER_MAX * n));
        std::vector<int> silent((size_t)sil_any * n);                 // [f][s]: stream s is still silent in frame f
        for (int f = 0; f < sil_any; f++) for (int s = 0; s < n; s++) silent[(size_t)f * n + s] = f < delay - b->fc[s];
        CK(cudaMemcpyAsync(b->d_mask, silent.data(), sizeof(int) * silent.size(), cudaMemcpyHostToDevice, st));
        CK(cudaStreamSynchronize(st));                              // (silent is a stack vector; this path runs at most FEATURES_DELAY times per reset)
        for (int f = sil_all; f < sil_any; f++) {
            if (copy_state(old, cur, SIGNAL | RNG, st)) return -1;
            if (launch_sample(b, pos0 + f, 1, spf, pcm + (size_t)f * spf, pcm_stride, f == 0 ? preload : 0, st, true)) return -1;
            restore_masked_kernel<<<n, 128, 0, st>>>(cur, old, b->d_mask + (size_t)f * n, SIGNAL | RNG, pcm + (size_t)f * spf, pcm_stride, spf);
            launches += 2;
        }
    }
    *live0 = sil_any;
    return launches;
}
// the launch that ends a batch's chunk: frames [live0, nf) of the frames at chunk positions [pos0, pos0 + nf), if any are left.
// Returns the number of engine kernels launched, < 0 on error.
static int launch_rest(LPCNetB200Batch *b, int pos0, int live0, int nf, int spf, short *pcm, long long pcm_stride, int preload, cudaStream_t st)
{
    if (nf <= live0) return 0;
    return launch_sample(b, pos0 + live0, nf - live0, spf, pcm + (size_t)live0 * spf, pcm_stride, live0 == 0 ? preload : 0, st, true) ? -1 : 1;
}
static int sample_frames(LPCNetB200Batch *b, int pos0, int nf, int spf, short *pcm, long long pcm_stride, int preload, cudaStream_t st)
{
    int sil_any = 0;
    int launches = sample_prefix(b, pos0, nf, spf, pcm, pcm_stride, preload, st, &sil_any);
    if (launches < 0) return -1;
    const int r = launch_rest(b, pos0, sil_any, nf, spf, pcm, pcm_stride, preload, st);
    if (r < 0) return -1;
    for (int &v : b->fc) v = std::min(1000, v + nf);
    return launches + r;
}

// The 100 Hz part of a chunk [c0, c0 + nf) of a call: the frame network on the batch's rows of the features; the chunk's last
// frame is what a tail reads.  Returns the number of engine kernels launched.
static int frame_chunk(LPCNetB200Batch *b, const float *d_feat, long long stream_stride, int frame_stride, int c0, int nf, cudaStream_t st)
{
    launch_frame_network(b->model, b->fs, d_feat + (size_t)c0 * frame_stride, stream_stride, frame_stride, b->n, nf, b->condA, b->condB, b->lpc_raw, st);
    b->cond_last = nf - 1;
    return frame_network_launches(b->model);
}

static int run_call(LPCNetB200Group *g, LPCNetB200Batch *b, const CallShape &c, const void *const *in, short *const *pcm, const PcmTarget *fwd,
                    int preload, cudaStream_t st);
// A batch call on device buffers: features or packets at d_in, PCM at d_pcm, everything on `st`
static int batch_call(LPCNetB200Batch *b, const CallShape &c, const void *d_in, short *d_pcm, int preload, cudaStream_t st)
{
    if (!b) { set_error("null batch"); return -1; }
    if (c.units <= 0) return 0;
    if (c.check()) return -1;
    if (preload < 0 || preload > c.spf) { set_error("preload must be in 0..samples_per_frame"); return -1; }
    if (c.decode && !b->model.codebooks) { set_error("decode: no VQ codebooks loaded (lpcnet_b200_batch_set_codebooks)"); return -1; }
    if (b->sink.dst && b->sink.pitch < c.pcm_samples()) {
        set_error("PCM sink pitch %lld smaller than the call's %lld samples per stream", b->sink.pitch, c.pcm_samples()); return -1;
    }
    return run_call(nullptr, b, c, &d_in, &d_pcm, b->sink.dst ? &b->sink : nullptr, preload, st);
}

int lpcnet_b200_batch_synthesize_device_ex(LPCNetB200Batch *b, const float *d_features, int nframes, int feature_stride,
                                           int samples_per_frame, short *d_pcm, int preload, void *cuda_stream)
{
    if (!b) { set_error("null batch"); return -1; }
    CK(cudaSetDevice(b->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : b->stream;
    int r = batch_call(b, CallShape::synthesis(nframes, feature_stride, samples_per_frame), d_features, d_pcm, preload, st);
    if (r == 0 && !cuda_stream) CK(cudaStreamSynchronize(st));
    return r;
}
int lpcnet_b200_batch_synthesize_device(LPCNetB200Batch *b, const float *d_features, int nframes, int feature_stride,
                                        int samples_per_frame, short *d_pcm, void *cuda_stream)
{
    return lpcnet_b200_batch_synthesize_device_ex(b, d_features, nframes, feature_stride, samples_per_frame, d_pcm, 0, cuda_stream);
}

int lpcnet_b200_batch_synthesize_ex(LPCNetB200Batch *b, const float *features, int nframes, int feature_stride,
                                    int samples_per_frame, short *pcm, int preload)
{
    if (!b) { set_error("null batch"); return -1; }
    if (nframes <= 0) return 0;
    if (!features || !pcm) { set_error("null buffer"); return -1; }
    CK(cudaSetDevice(b->device));
    const CallShape c = CallShape::synthesis(nframes, feature_stride, samples_per_frame);
    const size_t fbytes = c.in_bytes() * b->n, pbytes = sizeof(short) * c.pcm_samples() * b->n;
    if (ensure(b, (void **)&b->d_features, &b->d_features_cap, fbytes)) return -1;
    if (ensure(b, (void **)&b->d_pcm, &b->d_pcm_cap, pbytes)) return -1;
    if (order_enter(b, b->stream)) return -1;       // the staging buffers may still be read by work on another stream
    CK(cudaMemcpyAsync(b->d_features, features, fbytes, cudaMemcpyHostToDevice, b->stream));
    if (preload > 0)                                // teacher forcing reads the caller's signal from the output buffer (lpcnet.c:257)
        CK(cudaMemcpy2DAsync(b->d_pcm, c.pcm_samples() * sizeof(short), pcm, c.pcm_samples() * sizeof(short),
                             (size_t)std::min(preload, samples_per_frame) * sizeof(short), b->n, cudaMemcpyHostToDevice, b->stream));
    if (order_leave(b, b->stream)) return -1;
    if (batch_call(b, c, b->d_features, b->d_pcm, preload, b->stream)) return -1;
    CK(cudaMemcpyAsync(pcm, b->d_pcm, pbytes, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}
int lpcnet_b200_batch_synthesize(LPCNetB200Batch *b, const float *features, int nframes, int feature_stride,
                                 int samples_per_frame, short *pcm)
{
    return lpcnet_b200_batch_synthesize_ex(b, features, nframes, feature_stride, samples_per_frame, pcm, 0);
}

// ---- the reference's internal entry points around the same kernels (lpcnet_private.h:125-133), batched ----
// run_frame_network only (lpcnet.c:82-120): advances the 100 Hz state and the frame counters, keeps the conditioning of the LAST
// frame for lpcnet_b200_batch_synthesize_tail
int lpcnet_b200_batch_run_frame_network(LPCNetB200Batch *b, const float *features, int nframes, int feature_stride)
{
    if (!b) { set_error("null batch"); return -1; }
    if (nframes <= 0) return 0;
    if (!features || feature_stride < NB_FEAT) { set_error("run_frame_network: bad arguments"); return -1; }
    CK(cudaSetDevice(b->device));
    const size_t fbytes = sizeof(float) * (size_t)b->n * nframes * feature_stride;
    if (ensure(b, (void **)&b->d_features, &b->d_features_cap, fbytes)) return -1;
    if (order_enter(b, b->stream)) return -1;
    CK(cudaMemcpyAsync(b->d_features, features, fbytes, cudaMemcpyHostToDevice, b->stream));
    for (int c0 = 0; c0 < nframes; c0 += CHUNK) {
        const int nf = std::min(CHUNK, nframes - c0);
        frame_chunk(b, b->d_features, (long long)nframes * feature_stride, feature_stride, c0, nf, b->stream);
        for (int &v : b->fc) v = std::min(1000, v + nf);
    }
    if (order_leave(b, b->stream)) return -1;
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}

// lpcnet_synthesize_tail_impl (lpcnet.c:235-271): `samples` more samples with the conditioning of the last synthesize /
// run_frame_network call (zeros after a reset, what the snapshot held after a restore)
int lpcnet_b200_batch_synthesize_tail(LPCNetB200Batch *b, int samples, short *pcm, int preload)
{
    if (!b || !pcm || samples < 1 || samples > 65536) { set_error("synthesize_tail: bad arguments"); return -1; }
    if (preload < 0 || preload > samples) { set_error("preload must be in 0..samples"); return -1; }
    if (b->cond_last < 0) {
        set_error("synthesize_tail: a stream was imported since the last frame-network run and the exported state carries no conditioning; "
                  "call synthesize or run_frame_network first");
        return -1;
    }
    CK(cudaSetDevice(b->device));
    const size_t pbytes = sizeof(short) * (size_t)b->n * samples;
    if (ensure(b, (void **)&b->d_pcm, &b->d_pcm_cap, pbytes)) return -1;
    if (order_enter(b, b->stream)) return -1;
    if (preload > 0) CK(cudaMemcpyAsync(b->d_pcm, pcm, pbytes, cudaMemcpyHostToDevice, b->stream));
    b->kev_used = 0;
    // the frame counters were already advanced by the frame network run; the silent test of lpcnet.c:239 looks at the CURRENT
    // count, sample_frames() at the count before the frame: step back by one for the duration of the call
    std::vector<int> saved = b->fc;
    for (int &v : b->fc) v = v - 1;
    const int r = sample_frames(b, b->cond_last, 1, samples, b->d_pcm, samples, preload, b->stream);
    b->fc = saved;
    if (r < 0) return -1;
    b->last_launches = r;
    if (order_leave(b, b->stream)) return -1;
    CK(cudaMemcpyAsync(pcm, b->d_pcm, pbytes, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}

// run_frame_network_deferred / _flush (lpcnet.c:122-144): queue up to 4 feature frames without evaluating the network; the
// flush runs the frame network over each stream's queue (outputs discarded, state and frame counters advance).  As in the
// reference, a flush leaves the conditioning a tail reads as it was.
int lpcnet_b200_batch_frame_network_deferred(LPCNetB200Batch *b, const float *features, int feature_stride)
{
    if (!b || !features || feature_stride < NB_FEAT) { set_error("frame_network_deferred: bad arguments"); return -1; }
    const size_t fr = (size_t)b->n * NB_FEAT;
    b->deferred.resize(fr * DEFER_MAX);
    float *q = b->deferred.data();
    if (b->deferred_fill == DEFER_MAX) memmove(q, q + fr, sizeof(float) * fr * (DEFER_MAX - 1));
    else b->deferred_fill++;
    for (int &v : b->dfill) v = std::min(DEFER_MAX, v + 1);
    float *dst = q + fr * (b->deferred_fill - 1);
    for (int s = 0; s < b->n; s++) memcpy(dst + (size_t)s * NB_FEAT, features + (size_t)s * feature_stride, sizeof(float) * NB_FEAT);
    return 0;
}
int lpcnet_b200_batch_frame_network_flush(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return -1; }
    const int F = b->deferred_fill, n = b->n;
    const std::vector<int> fill = b->dfill;
    b->deferred_fill = 0;
    std::fill(b->dfill.begin(), b->dfill.end(), 0);
    // stream s runs queued frame k iff k >= F - fill[s]; from frame k_all on every stream does
    int k0 = F, k_all = 0;
    for (int v : fill) { k0 = std::min(k0, F - v); k_all = std::max(k_all, F - v); }
    if (k0 >= F) return 0;
    CK(cudaSetDevice(b->device));
    const size_t fr = (size_t)n * NB_FEAT;
    std::vector<float> f((size_t)n * F * NB_FEAT);                   // [n][F][20]
    std::vector<int> keep((size_t)F * n);                            // [F][n]
    for (int k = 0; k < F; k++) for (int s = 0; s < n; s++) {
        memcpy(&f[((size_t)s * F + k) * NB_FEAT], b->deferred.data() + fr * k + (size_t)s * NB_FEAT, sizeof(float) * NB_FEAT);
        keep[(size_t)k * n + s] = k < F - fill[s];
    }
    if (ensure(b, (void **)&b->d_features, &b->d_features_cap, sizeof(float) * f.size())) return -1;
    if (k_all > k0) {
        if (!alloc_state(shadow_fields(b), FRAME)) { set_error("flush: device allocation failed"); return -1; }
        if (!b->d_mask) CK(cudaMalloc((void **)&b->d_mask, sizeof(int) * DEFER_MAX * n));
    }
    cudaStream_t st = b->stream;
    if (order_enter(b, st)) return -1;
    CK(cudaMemcpyAsync(b->d_features, f.data(), sizeof(float) * f.size(), cudaMemcpyHostToDevice, st));
    if (k_all > k0) CK(cudaMemcpyAsync(b->d_mask, keep.data(), sizeof(int) * keep.size(), cudaMemcpyHostToDevice, st));
    if (park_tail(b, st)) return -1;
    // frames only some streams run: one launch per frame, the others' 100 Hz state put back after it (vq_mem too, which the
    // frame network does not write: putting it back changes nothing)
    const Fields cur = batch_fields(b, -1), old = shadow_fields(b);
    for (int k = k0; k < k_all; k++) {
        if (copy_state(old, cur, FRAME, st)) return -1;
        launch_frame_network(b->model, b->fs, b->d_features + (size_t)k * NB_FEAT, (long long)F * NB_FEAT, NB_FEAT, n, 1, b->condA, b->condB, b->lpc_raw, st);
        restore_masked_kernel<<<n, 128, 0, st>>>(cur, old, b->d_mask + (size_t)k * n, FRAME, nullptr, 0, 0);
    }
    if (k_all < F)
        launch_frame_network(b->model, b->fs, b->d_features + (size_t)k_all * NB_FEAT, (long long)F * NB_FEAT, NB_FEAT, n, F - k_all, b->condA, b->condB, b->lpc_raw, st);
    CK(cudaGetLastError());
    for (int s = 0; s < n; s++) b->fc[s] = std::min(1000, b->fc[s] + fill[s]);
    if (order_leave(b, st)) return -1;
    CK(cudaStreamSynchronize(st));                                   // (f and keep are read by the copies above)
    return 0;
}

int lpcnet_b200_batch_decode_device(LPCNetB200Batch *b, const unsigned char *d_packets, int npackets, short *d_pcm, void *cuda_stream)
{
    if (!b) { set_error("null batch"); return -1; }
    if (npackets <= 0) return 0;
    CK(cudaSetDevice(b->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : b->stream;
    int r = batch_call(b, CallShape::packets(npackets), d_packets, d_pcm, 0, st);
    if (r == 0 && !cuda_stream) CK(cudaStreamSynchronize(st));
    return r;
}

int lpcnet_b200_batch_decode(LPCNetB200Batch *b, const unsigned char *packets, int npackets, short *pcm)
{
    if (!b) { set_error("null batch"); return -1; }
    if (npackets <= 0) return 0;
    if (!packets || !pcm) { set_error("null buffer"); return -1; }
    CK(cudaSetDevice(b->device));
    const CallShape c = CallShape::packets(npackets);
    const size_t kbytes = c.in_bytes() * b->n, pbytes = sizeof(short) * c.pcm_samples() * b->n;
    if (ensure(b, (void **)&b->d_packets, &b->d_packets_cap, kbytes)) return -1;
    if (ensure(b, (void **)&b->d_pcm, &b->d_pcm_cap, pbytes)) return -1;
    if (order_enter(b, b->stream)) return -1;
    CK(cudaMemcpyAsync(b->d_packets, packets, kbytes, cudaMemcpyHostToDevice, b->stream));
    if (order_leave(b, b->stream)) return -1;
    if (batch_call(b, c, b->d_packets, b->d_pcm, 0, b->stream)) return -1;
    CK(cudaMemcpyAsync(pcm, b->d_pcm, pbytes, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}

float lpcnet_b200_batch_last_sample_kernel_ms(const LPCNetB200Batch *b, int *launches)
{
    if (!b) return 0.f;
    if (launches) *launches = b->last_launches;
    return timed_ms(b->kev, b->kev_used);
}

// ---- groups: the synthesize / decode calls of several batches of one flavour and GRU_A size on one device as one call ----
// Each chunk runs every member's 100 Hz part and silent-frame prefix with the member's own launches, then ONE per-sample launch
// for the frames that remain (GroupSampleParams; sample_kernel.cu, sample_kernel_f32.cu, sample_kernel_f32n.cu).  The members
// keep all their state and host mirrors; the group only holds the launch plan, a stream and staging for its host-pointer calls and
// the event timers of its launches.
struct LPCNetB200Group {
    int count, device, na, n_total;
    LPCNetB200Batch *m[GROUP_MAX];
    bool is_float;                    // the members' flavour
    bool neuron;                      // float: the neuron-per-lane kernel (group_plan_float)
    int spc, slots, ctas;             // the launch plan (group_plan, group_plan_float): slots = streams a CTA lays out
    bool fast_cvt;                    // conversion-free rounding: only if every member allows it
    uint32_t smem_bytes;              // largest shared-memory footprint of the members
    cudaStream_t stream;
    std::vector<cudaEvent_t> kev;     // event pairs around the group's own per-sample launches of the last call
    int kev_used, last_launches;
    PcmForwarder fwd;                 // PCM forwarded to the targets of group_call
    void *d_in; size_t d_in_cap;      // staging of the host-pointer calls
    short *d_pcm; size_t d_pcm_cap;
};

int lpcnet_b200_debug_group_plan(const int *n, int count, int sms, int override_spc, int *spc, int *ctas)
{
    if (!n || count < 1 || count > GROUP_MAX || sms < 1 || !spc || !ctas) { set_error("debug_group_plan: bad arguments"); return -1; }
    for (int k = 0; k < count; k++) if (n[k] < 1) { set_error("debug_group_plan: member %d has no streams", k); return -1; }
    *spc = group_plan(n, count, sms, override_spc, ctas);
    return 0;
}

static int plan_ctas(const int *n, int count, int slots)
{
    int c = 0;
    for (int k = 0; k < count; k++) c += (n[k] + slots - 1) / slots;
    return c;
}
static bool group_plan_float(const int *n, int count, int sms, int override_spc, bool lane_stream, int *spc, int *slots, int *ctas)
{
    bool neuron;
    *spc = group_plan(n, count, sms, override_spc, ctas);
    *slots = float_slots(*spc, lane_stream, &neuron);
    *ctas = plan_ctas(n, count, *slots);
    return neuron;
}

int lpcnet_b200_debug_group_plan_float(const int *n, int count, int sms, int override_spc, int lane_stream, int *spc, int *slots, int *ctas)
{
    if (!n || count < 1 || count > GROUP_MAX || sms < 1 || !spc || !slots || !ctas) { set_error("debug_group_plan_float: bad arguments"); return -1; }
    for (int k = 0; k < count; k++) if (n[k] < 1) { set_error("debug_group_plan_float: member %d has no streams", k); return -1; }
    return group_plan_float(n, count, sms, override_spc, lane_stream != 0, spc, slots, ctas) ? 1 : 0;
}

int lpcnet_b200_debug_mixed_plan(const int *n, const int *na, const int *is_float, int count, int sms, int override_spc, int lane_stream,
                                 int *spc, int *class_of, int *class_ctas, int *class_neuron)
{
    if (!n || !na || !is_float || count < 1 || count > GROUP_MAX || sms < 1 || !spc || !class_of || !class_ctas || !class_neuron) {
        set_error("debug_mixed_plan: bad arguments"); return -1;
    }
    for (int k = 0; k < count; k++) {
        if (n[k] < 1) { set_error("debug_mixed_plan: member %d has no streams", k); return -1; }
        if (!na_supported(na[k])) { set_error("debug_mixed_plan: member %d has %d GRU_A units (128, 256 or 384)", k, na[k]); return -1; }
        if (is_float[k] != 0 && is_float[k] != 1) { set_error("debug_mixed_plan: member %d: is_float must be 0 or 1", k); return -1; }
    }
    bool neuron[GROUP_MAX];
    const int classes = mixed_plan(n, na, is_float, count, sms, override_spc, lane_stream != 0, spc, class_of, class_ctas, neuron);
    for (int c = 0; c < classes; c++) class_neuron[c] = neuron[c] ? 1 : 0;
    return classes;
}

void lpcnet_b200_group_destroy(LPCNetB200Group *g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    if (g->stream) { cudaStreamSynchronize(g->stream); cudaStreamDestroy(g->stream); }
    g->fwd.destroy();
    if (g->d_in) cudaFree(g->d_in);
    if (g->d_pcm) cudaFree(g->d_pcm);
    for (cudaEvent_t e : g->kev) cudaEventDestroy(e);
    delete g;
}

LPCNetB200Group *lpcnet_b200_group_create(LPCNetB200Batch *const *batches, int count)
{
    if (group_members_check(batches, count, "group_create", true)) return nullptr;
    int n[GROUP_MAX], ctas;
    for (int k = 0; k < count; k++) n[k] = batches[k]->n;
    const char *e = getenv("LPCNET_B200_STREAMS_PER_CTA");
    return group_init(batches, count, group_plan(n, count, device_sms(batches[0]->device), e ? atoi(e) : 0, &ctas));
}

int lpcnet_b200_group_streams(const LPCNetB200Group *g) { return g ? g->n_total : 0; }

// the fused launch over the members that still have frames [live0[k], nf) of the chunk to run
static int launch_group(LPCNetB200Group *g, const int *live0, int nf, int spf, short *const *pcm, long long pcm_stride, cudaStream_t st)
{
    GroupSampleParams gp = {};
    int ctas = 0;
    for (int k = 0; k < g->count; k++) {
        LPCNetB200Batch *b = g->m[k];
        if (live0[k] >= nf) continue;
        SampleParams &p = gp.m[gp.count];
        p = sample_params(b, live0[k], nf - live0[k], spf, pcm[k] + (size_t)live0[k] * spf, pcm_stride);
        p.spc = g->spc;
        p.one_half = g->spc <= HALF;
        p.fast_cvt = g->fast_cvt ? 1 : 0;
        if (g->neuron) { p.L = b->model.Ln; p.image = b->model.image_n; }     // the member's neuron-per-lane layout and image
        gp.cta0[gp.count++] = ctas;
        ctas += (b->n + g->slots - 1) / g->slots;
    }
    if (!gp.count) return 0;
    if (time_launch(g->kev, &g->kev_used, st)) return -1;
    cudaError_t e;
#define LPCNET_GROUP_DISPATCH(ns) (!g->is_float ? ns::launch_group_sample_kernel(gp, ctas, g->smem_bytes, st) \
                                   : g->neuron ? ns::launch_group_sample_kernel_f32n(gp, ctas, g->smem_bytes, st) \
                                               : ns::launch_group_sample_kernel_f32(gp, ctas, g->smem_bytes, st))
    switch (g->na) {
    case 128: e = LPCNET_GROUP_DISPATCH(na128); break;
    case 256: e = LPCNET_GROUP_DISPATCH(na256); break;
    default:  e = LPCNET_GROUP_DISPATCH(na384); break;
    }
#undef LPCNET_GROUP_DISPATCH
    if (e != cudaSuccess) { set_error("group per-sample kernel launch failed: %s", cudaGetErrorString(e)); return -1; }
    if (time_launch(g->kev, &g->kev_used, st)) return -1;
    return 1;
}

// Core of the batch and group calls (g NULL: a call of batch b alone, with its preload; else of the group's members, preload 0).
// Member k reads in[k] (features [n_k][frames][stride], or packets that are first decoded into the member's feature staging) and
// writes pcm[k] ([n_k][frames * spf]), all device pointers, everything on `st`.  Per chunk: every member's frame network and
// silent prefix, then the launch that ends the chunk (the batch's own, or one for the whole group), and the chunk's PCM forwarded
// to fwd[k] for the members that have a target (fwd NULL: none).
static int run_call(LPCNetB200Group *g, LPCNetB200Batch *b, const CallShape &c, const void *const *in, short *const *pcm, const PcmTarget *fwd,
                    int preload, cudaStream_t st)
{
    LPCNetB200Batch *const *m = g ? g->m : &b;
    const int count = g ? g->count : 1, nframes = c.frames(), spf = c.spf;
    const long long stream_stride = (long long)nframes * c.stride, pcm_stride = c.pcm_samples();
    const float *feat[GROUP_MAX];
    if (c.decode) {
        for (int k = 0; k < count; k++)
            if (ensure(m[k], (void **)&m[k]->d_features, &m[k]->d_features_cap, sizeof(float) * (size_t)m[k]->n * stream_stride)) return -1;
        for (int k = 0; k < count; k++) {
            if (order_enter(m[k], st)) return -1;
            launch_decode_packets(m[k]->model, m[k]->fs, (const uint8_t *)in[k], m[k]->n, c.units, m[k]->d_features, st);
            if (order_leave(m[k], st)) return -1;
        }
    }
    for (int k = 0; k < count; k++) feat[k] = c.decode ? m[k]->d_features : (const float *)in[k];
    PcmForwarder &fw = g ? g->fwd : b->fwd;
    bool forwarding = false;
    for (int k = 0; fwd && k < count; k++) forwarding = forwarding || fwd[k].dst;
    if (forwarding && fw.open()) return -1;
    int launches = 0;
    if (g) g->kev_used = 0;
    for (int k = 0; k < count; k++) {
        m[k]->kev_used = 0;
        if (order_enter(m[k], st)) return -1;
    }
    for (int c0 = 0; c0 < nframes; c0 += CHUNK) {
        const int nf = std::min(CHUNK, nframes - c0), pre = c0 == 0 ? preload : 0;
        int live0[GROUP_MAX];
        short *pc[GROUP_MAX];
        for (int k = 0; k < count; k++) {
            pc[k] = pcm[k] + (size_t)c0 * spf;
            launches += frame_chunk(m[k], feat[k], stream_stride, c.stride, c0, nf, st);
            const int r = sample_prefix(m[k], 0, nf, spf, pc[k], pcm_stride, pre, st, &live0[k]);
            if (r < 0) return -1;
            launches += r;
        }
        const int r = g ? launch_group(g, live0, nf, spf, pc, pcm_stride, st) : launch_rest(b, 0, live0[0], nf, spf, pc[0], pcm_stride, pre, st);
        if (r < 0) return -1;
        launches += r;
        for (int k = 0; k < count; k++) for (int &v : m[k]->fc) v = std::min(1000, v + nf);
        for (int k = 0; forwarding && k < count; k++)
            if (fwd[k].dst && fw.forward_to_sink(fwd[k], m[k]->n, pcm[k], pcm_stride, c0, nf, spf, st)) return -1;
    }
    CK(cudaGetLastError());
    if (forwarding && fw.join(st)) return -1;
    for (int k = 0; k < count; k++) if (order_leave(m[k], st)) return -1;
    (g ? g->last_launches : b->last_launches) = launches + (c.decode ? count : 0);    // (+ the packet decoders)
    return 0;
}

// What a public group call refuses, in this order: a NULL group, a member with a PCM sink, NULL buffers, a bad shape, a decode
// with a member without codebooks.  Returns 1 for a call without units: nothing to do.
static int group_entry(LPCNetB200Group *g, const CallShape &c, const void *in, const void *out)
{
    if (group_check(g, CallShape{}, true)) return -1;
    CK(cudaSetDevice(g->device));
    if (c.units <= 0) return 1;
    if (!in || !out) { set_error("null buffer"); return -1; }
    return group_check(g, c, false);
}
// a checked call on device buffers of the group's rows
static int group_call_rows(LPCNetB200Group *g, const CallShape &c, const void *in, short *pcm, cudaStream_t st)
{
    const void *pin[GROUP_MAX]; short *ppcm[GROUP_MAX];
    group_rows(g, c, in, pcm, nullptr, pin, ppcm);
    return group_call(g, c, pin, ppcm, nullptr, st);
}
static int group_device(LPCNetB200Group *g, const CallShape &c, const void *d_in, short *d_pcm, void *cuda_stream)
{
    const int r = group_entry(g, c, d_in, d_pcm);
    if (r) return r < 0 ? -1 : 0;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : g->stream;
    if (group_call_rows(g, c, d_in, d_pcm, st)) return -1;
    if (!cuda_stream) CK(cudaStreamSynchronize(st));
    return 0;
}
// host-pointer calls: the rows go through the group's own staging buffers on its stream; returns once the PCM is on the host
static int group_host(LPCNetB200Group *g, const CallShape &c, const void *in, short *pcm)
{
    const int r = group_entry(g, c, in, pcm);
    if (r) return r < 0 ? -1 : 0;
    const size_t in_bytes = c.in_bytes() * g->n_total, pcm_bytes = sizeof(short) * c.pcm_samples() * g->n_total;
    // (earlier host calls are complete and `_device` calls never touch these buffers: nothing can still be using them)
    if (grow_buffer(&g->d_in, &g->d_in_cap, in_bytes) || grow_buffer((void **)&g->d_pcm, &g->d_pcm_cap, pcm_bytes)) return -1;
    CK(cudaMemcpyAsync(g->d_in, in, in_bytes, cudaMemcpyHostToDevice, g->stream));
    if (group_call_rows(g, c, g->d_in, g->d_pcm, g->stream)) return -1;
    CK(cudaMemcpyAsync(pcm, g->d_pcm, pcm_bytes, cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return 0;
}

int lpcnet_b200_group_synthesize_device(LPCNetB200Group *g, const float *d_features, int nframes, int feature_stride,
                                        int samples_per_frame, short *d_pcm, void *cuda_stream)
{
    return group_device(g, CallShape::synthesis(nframes, feature_stride, samples_per_frame), d_features, d_pcm, cuda_stream);
}
int lpcnet_b200_group_synthesize(LPCNetB200Group *g, const float *features, int nframes, int feature_stride,
                                 int samples_per_frame, short *pcm)
{
    return group_host(g, CallShape::synthesis(nframes, feature_stride, samples_per_frame), features, pcm);
}
int lpcnet_b200_group_decode_device(LPCNetB200Group *g, const unsigned char *d_packets, int npackets, short *d_pcm, void *cuda_stream)
{
    return group_device(g, CallShape::packets(npackets), d_packets, d_pcm, cuda_stream);
}
int lpcnet_b200_group_decode(LPCNetB200Group *g, const unsigned char *packets, int npackets, short *pcm)
{
    return group_host(g, CallShape::packets(npackets), packets, pcm);
}

}  // extern "C"

// ---- the parts of group_create that mixed groups share (engine.h) ----
int lpcnet_b200::group_members_check(LPCNetB200Batch *const *batches, int count, const char *who, bool one_shape)
{
    if (!batches || count < 1 || count > GROUP_MAX) { set_error("%s: 1..%d member batches", who, GROUP_MAX); return -1; }
    for (int k = 0; k < count; k++) {
        const LPCNetB200Batch *b = batches[k];
        if (!b) { set_error("%s: member %d is NULL", who, k); return -1; }
        if (one_shape && b->model.is_float != batches[0]->model.is_float) {
            set_error("%s: member %d holds %s model, member 0 %s one; the members of a group are all int8 or all float", who, k,
                      b->model.is_float ? "a float" : "an int8", batches[0]->model.is_float ? "a float" : "an int8");
            return -1;
        }
        if (b->device != batches[0]->device) { set_error("%s: member %d is on device %d, member 0 on device %d", who, k, b->device, batches[0]->device); return -1; }
        if (one_shape && b->model.na != batches[0]->model.na) { set_error("%s: member %d has %d GRU_A units, member 0 has %d", who, k, b->model.na, batches[0]->model.na); return -1; }
        for (int j = 0; j < k; j++) if (batches[j] == b) { set_error("%s: member %d is listed twice (also member %d)", who, k, j); return -1; }
    }
    return 0;
}

int lpcnet_b200::device_sms(int device)
{
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 132;
    return sms;
}

int lpcnet_b200::batch_device(const LPCNetB200Batch *b) { return b->device; }

LPCNetB200Group *lpcnet_b200::group_init(LPCNetB200Batch *const *batches, int count, int spc)
{
    if (cudaSetDevice(batches[0]->device) != cudaSuccess) { set_error("group_create: cudaSetDevice(%d) failed", batches[0]->device); return nullptr; }
    LPCNetB200Group *g = new LPCNetB200Group();
    g->count = count; g->device = batches[0]->device; g->na = batches[0]->model.na;
    g->is_float = batches[0]->model.is_float != 0;
    g->fast_cvt = true;
    int n[GROUP_MAX];
    for (int k = 0; k < count; k++) {
        LPCNetB200Batch *b = batches[k];
        g->m[k] = b; n[k] = b->n; g->n_total += b->n;
        g->fast_cvt = g->fast_cvt && batch_fast_cvt(b);
    }
    g->spc = spc;
    g->slots = g->is_float ? float_slots(spc, getenv("LPCNET_B200_FLOAT_LANE_STREAM") != nullptr, &g->neuron) : spc;
    g->ctas = plan_ctas(n, count, g->slots);
    for (int k = 0; k < count; k++)      // the footprint of the layout the chosen kernel uses
        g->smem_bytes = std::max(g->smem_bytes, g->neuron ? batches[k]->model.Ln.total_bytes : batches[k]->model.L.total_bytes);
    if (cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking) != cudaSuccess) {
        set_error("group_create: cudaStreamCreate failed"); lpcnet_b200_group_destroy(g); return nullptr;
    }
    return g;
}

int lpcnet_b200::mixed_plan(const int *n, const int *na, const int *is_float, int count, int sms, int override_spc, bool lane_stream,
                            int *spc, int *class_of, int *class_ctas, bool *class_neuron)
{
    int ctas, classes = 0, cls_na[GROUP_MAX], cls_float[GROUP_MAX], slots[GROUP_MAX];
    *spc = group_plan(n, count, sms, override_spc, &ctas);
    for (int k = 0; k < count; k++) {
        int c = 0;
        while (c < classes && (cls_na[c] != na[k] || cls_float[c] != is_float[k])) c++;
        if (c == classes) {
            cls_na[c] = na[k]; cls_float[c] = is_float[k]; class_ctas[c] = 0; class_neuron[c] = false;
            slots[c] = is_float[k] ? float_slots(*spc, lane_stream, &class_neuron[c]) : *spc;
            classes++;
        }
        class_of[k] = c;
        class_ctas[c] += (n[k] + slots[c] - 1) / slots[c];
    }
    return classes;
}

int lpcnet_b200::group_check(const LPCNetB200Group *g, const CallShape &c, bool refuse_sinks)
{
    if (!g) { set_error("null group"); return -1; }
    for (int k = 0; refuse_sinks && k < g->count; k++)
        if (g->m[k]->sink.dst) { set_error("group call: member %d has a PCM sink set; groups do not forward PCM to sinks", k); return -1; }
    if (c.units <= 0) return 0;
    if (c.check()) return -1;
    for (int k = 0; c.decode && k < g->count; k++)
        if (!g->m[k]->model.codebooks) { set_error("group decode: member %d has no VQ codebooks loaded (lpcnet_b200_batch_set_codebooks)", k); return -1; }
    return 0;
}

void lpcnet_b200::group_rows(const LPCNetB200Group *g, const CallShape &c, const void *in, short *pcm, const int *rows, const void **pin, short **ppcm)
{
    for (int k = 0, row = 0; k < g->count; row += g->m[k]->n, k++) {
        const size_t r = rows ? rows[k] : row;
        pin[k] = (const char *)in + c.in_bytes() * r;
        ppcm[k] = pcm + c.pcm_samples() * r;
    }
}

int lpcnet_b200::group_call(LPCNetB200Group *g, const CallShape &c, const void *const *in, short *const *pcm, const PcmTarget *fwd, cudaStream_t st)
{
    return run_call(g, nullptr, c, in, pcm, fwd, 0, st);
}

extern "C" {

// the group's fused launches plus the members' own launches for their silent-frame prefixes, in the last group call (the
// latter until the member's next call)
float lpcnet_b200_group_last_sample_kernel_ms(const LPCNetB200Group *g, int *launches)
{
    if (!g) return 0.f;
    if (launches) *launches = g->last_launches;
    if (cudaSetDevice(g->device) != cudaSuccess) return -1.f;
    float total = timed_ms(g->kev, g->kev_used);
    for (int k = 0; k < g->count && total >= 0.f; k++) {
        const float ms = timed_ms(g->m[k]->kev, g->m[k]->kev_used);
        total = ms < 0.f ? -1.f : total + ms;
    }
    return total;
}

// ---- PCM sink: the multi-GPU gather as part of the call (SURVEY 8e: the only exchange of the path) ----
int lpcnet_b200_batch_set_pcm_sink(LPCNetB200Batch *b, short *sink, long long pitch_samples, long long first_row)
{
    if (!b) { set_error("null batch"); return -1; }
    CK(cudaSetDevice(b->device));
    if (order_sync(b)) return -1;
    if (b->fwd.stream) CK(cudaStreamSynchronize(b->fwd.stream));
    b->sink = PcmTarget{sink, pitch_samples, first_row};
    return 0;
}
int lpcnet_b200_ipc_export(void *d_ptr, unsigned char handle[64])
{
    cudaIpcMemHandle_t h;
    static_assert(sizeof(h) == 64, "CUDA IPC handle size");
    CK(cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle, &h, 64);
    return 0;
}
void *lpcnet_b200_ipc_open(const unsigned char handle[64])
{
    cudaIpcMemHandle_t h; memcpy(&h, handle, 64);
    void *p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { set_error("cudaIpcOpenMemHandle: %s", cudaGetErrorString(cudaGetLastError())); return nullptr; }
    return p;
}
int lpcnet_b200_ipc_close(void *p) { CK(cudaIpcCloseMemHandle(p)); return 0; }

// CUDA-event stopwatch on the engine's own stream (the stream every engine kernel is launched on when the caller
// passes cuda_stream == NULL): start records an event, stop records another, synchronises and returns the ms between.
int lpcnet_b200_batch_timer_start(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return -1; }
    CK(cudaSetDevice(b->device));
    CK(cudaEventRecord(b->ev0, b->stream));
    return 0;
}
float lpcnet_b200_batch_timer_stop(LPCNetB200Batch *b)
{
    if (!b) return -1.f;
    float ms = 0.f;
    if (cudaEventRecord(b->ev1, b->stream) != cudaSuccess || cudaEventSynchronize(b->ev1) != cudaSuccess ||
        cudaEventElapsedTime(&ms, b->ev0, b->ev1) != cudaSuccess) { set_error("timer: %s", cudaGetErrorString(cudaGetLastError())); return -1.f; }
    return ms;
}
// Evict L2 between timed iterations: overwrite a scratch buffer larger than the 126 MB L2 on the engine's stream.
int lpcnet_b200_batch_flush_l2(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return -1; }
    static void *scratch[64] = {nullptr};
    const size_t bytes = 256u << 20;
    CK(cudaSetDevice(b->device));
    if (b->device < 0 || b->device >= 64) { set_error("flush_l2: device index"); return -1; }
    if (!scratch[b->device]) CK(cudaMalloc(&scratch[b->device], bytes));
    CK(cudaMemsetAsync(scratch[b->device], 0x5a, bytes, b->stream));
    return 0;
}
int lpcnet_b200_batch_sync(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return -1; }
    CK(cudaSetDevice(b->device));
    if (order_sync(b)) return -1;
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}
// Device memory helpers so that a plain-C / ctypes caller can keep inputs resident in HBM (no torch needed).
void *lpcnet_b200_device_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { set_error("cudaMalloc(%zu) failed", bytes); return nullptr; }
    return p;
}
void lpcnet_b200_device_free(void *p) { if (p) cudaFree(p); }
// (from pageable memory cudaMemcpy may return before the DMA has landed; the synchronise makes the data visible to work on any stream)
int lpcnet_b200_memcpy_h2d(void *dst, const void *src, size_t bytes) { CK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); CK(cudaStreamSynchronize(0)); return 0; }
int lpcnet_b200_memcpy_d2h(void *dst, const void *src, size_t bytes) { CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost)); return 0; }
int lpcnet_b200_set_device(int device) { CK(cudaSetDevice(device)); return 0; }
// CUDA streams for callers without their own CUDA binding (the `cuda_stream` argument of the `_device` entry points)
void *lpcnet_b200_stream_create(void)
{
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) { set_error("cudaStreamCreate failed"); return nullptr; }
    return s;
}
void lpcnet_b200_stream_destroy(void *s) { if (s) cudaStreamDestroy((cudaStream_t)s); }
int lpcnet_b200_stream_sync(void *s) { CK(cudaStreamSynchronize((cudaStream_t)s)); return 0; }

int lpcnet_b200_batch_algorithmic_bytes(const LPCNetB200Batch *b, long *total, long *sparse_gemv)
{
    if (!b) { set_error("null batch"); return -1; }
    if (total) *total = b->model.algo_bytes_total;
    if (sparse_gemv) *sparse_gemv = b->model.algo_bytes_sparse;
    return 0;
}

// ---- state by value (what the PLC does with `LPCNetState copy = *st`, lpcnet_plc.c:216-230): one stream <-> host blob ----
int lpcnet_b200_batch_state_size(const LPCNetB200Batch *b)
{
    return b ? state_words(b->model.na) * 4 : -1;
}
// stream s's record without the tail part <-> host buffer `rec`, through the staging buffer.  unpack: rec -> stream.
static int stream_record(LPCNetB200Batch *b, int s, void *rec, bool unpack)
{
    CK(cudaSetDevice(b->device));
    const Fields t = batch_fields(b, -1);
    const int words = record_words(t, F_COND_A);
    const size_t bytes = sizeof(float) * words;
    if (ensure(b, (void **)&b->d_state, &b->d_state_cap, bytes)) return -1;
    if (order_enter(b, b->stream)) return -1;
    if (unpack) {
        CK(cudaMemcpyAsync(b->d_state, rec, bytes, cudaMemcpyHostToDevice, b->stream));
        records_kernel<true><<<1, 128, 0, b->stream>>>(t, nullptr, s, b->d_state, words, STATE);
    } else {
        records_kernel<false><<<1, 128, 0, b->stream>>>(t, nullptr, s, b->d_state, words, STATE);
        CK(cudaMemcpyAsync(rec, b->d_state, bytes, cudaMemcpyDeviceToHost, b->stream));
    }
    if (order_leave(b, b->stream)) return -1;
    CK(cudaStreamSynchronize(b->stream));
    return 0;
}
static int state_move(LPCNetB200Batch *b, int s, void *buf, int dir)
{
    if (!b || !buf || s < 0 || s >= b->n) { set_error("state export/import: bad arguments"); return -1; }
    if (!dir && b->dfill[s] > 0) {
        set_error("export_state: stream %d has %d queued frames and the exported state has no room for them; flush first", s, b->dfill[s]);
        return -1;
    }
    if (stream_record(b, s, buf, dir)) return -1;
    if (dir) {
        int fcv; memcpy(&fcv, (const char *)buf + sizeof(float) * record_words(batch_fields(b, -1), F_FRAME_COUNT), sizeof(fcv));
        b->fc[s] = fcv;
        b->dfill[s] = 0;
        b->cond_last = -1;          // the blob carries no conditioning: no tail until the next frame-network run
    }
    return 0;
}
int lpcnet_b200_batch_export_state(LPCNetB200Batch *b, int s, void *buf) { return state_move(b, s, buf, 0); }
int lpcnet_b200_batch_import_state(LPCNetB200Batch *b, int s, const void *buf) { return state_move(b, s, const_cast<void *>(buf), 1); }

// fields of stream s's record; misc = {last_exc, frame counter (from the host mirror)}
int lpcnet_b200_batch_get_state(LPCNetB200Batch *b, int s, float *gru_a, float *gru_b, float *last_sig, int *misc, uint32_t *rng)
{
    if (!b || s < 0 || s >= b->n) { set_error("bad stream index"); return -1; }
    const Fields t = batch_fields(b, -1);
    std::vector<float> rec(record_words(t, F_COND_A));
    if (stream_record(b, s, rec.data(), false)) return -1;
    auto pick = [&](void *dst, int j) { if (dst) memcpy(dst, &rec[record_words(t, j)], sizeof(float) * t.f[j].planes * t.f[j].width); };
    pick(gru_a, F_HA); pick(gru_b, F_HB); pick(last_sig, F_LAST_SIG); pick(misc, F_LAST_EXC); pick(rng, F_RNG);
    if (misc) misc[1] = b->fc[s];
    return 0;
}

// ---- whole streams between batches on the device (compaction, shard rebalancing, cloning) ----
// Each batch's staging buffer d_state holds [count] source rows, [count] destination rows, then the count records (in the order of state_fields).
// The records are packed on src's stream, copied into dst's staging (peer DMA across devices) and unpacked on dst's stream;
// staging makes src == dst read every record before any is written.
static int copy_check(const LPCNetB200Batch *dst, const int *dst_rows, const LPCNetB200Batch *src, const int *src_rows, int count)
{
    if (!dst || !dst_rows || !src || !src_rows || count < 0) { set_error("copy_streams: bad arguments"); return -1; }
    if (dst->model.na != src->model.na) { set_error("copy_streams: dst has %d GRU_A units, src %d", dst->model.na, src->model.na); return -1; }
    if (dst->model.is_float != src->model.is_float) { set_error("copy_streams: one batch holds an int8 model, the other a float model"); return -1; }
    const ModelConfig &a = dst->model.cfg, &c = src->model.cfg;
    if (a.features_delay != c.features_delay || a.end2end != c.end2end || a.lpc_gamma != c.lpc_gamma) {
        set_error("copy_streams: model switches differ (FEATURES_DELAY %d / %d, END2END %d / %d, LPC_GAMMA %g / %g)",
                  a.features_delay, c.features_delay, a.end2end, c.end2end, (double)a.lpc_gamma, (double)c.lpc_gamma);
        return -1;
    }
    std::vector<char> seen(dst->n, 0);
    for (int k = 0; k < count; k++) {
        if (src_rows[k] < 0 || src_rows[k] >= src->n) { set_error("copy_streams: source row %d out of range (%d streams)", src_rows[k], src->n); return -1; }
        if (dst_rows[k] < 0 || dst_rows[k] >= dst->n) { set_error("copy_streams: destination row %d out of range (%d streams)", dst_rows[k], dst->n); return -1; }
        if (seen[dst_rows[k]]) { set_error("copy_streams: destination row %d listed twice", dst_rows[k]); return -1; }
        seen[dst_rows[k]] = 1;
    }
    return 0;
}

int lpcnet_b200_batch_copy_streams(LPCNetB200Batch *dst, const int *dst_rows, LPCNetB200Batch *src, const int *src_rows, int count)
{
    if (copy_check(dst, dst_rows, src, src_rows, count)) return -1;
    if (count == 0) return 0;
    const bool tails = dst->cond_last >= 0 && src->cond_last >= 0;      // else dst refuses tails until its next frame-network run
    const Fields ts = batch_fields(src, tails ? src->cond_last : -1), td = batch_fields(dst, tails ? dst->cond_last : -1);
    const unsigned parts = tails ? ALL : STATE;
    const int words = record_words(ts, NFIELDS);
    const size_t rows_bytes = sizeof(int) * 2 * (size_t)count, bytes = rows_bytes + sizeof(float) * (size_t)count * words;
    std::vector<int> rows(2 * (size_t)count);
    std::copy(src_rows, src_rows + count, rows.begin());
    std::copy(dst_rows, dst_rows + count, rows.begin() + count);
    CK(cudaSetDevice(src->device));
    if (ensure(src, (void **)&src->d_state, &src->d_state_cap, bytes)) return -1;
    CK(cudaSetDevice(dst->device));
    if (ensure(dst, (void **)&dst->d_state, &dst->d_state_cap, bytes)) return -1;

    // 1. pack on src's stream
    CK(cudaSetDevice(src->device));
    int *s_rows = reinterpret_cast<int *>(src->d_state);
    float *s_rec = reinterpret_cast<float *>(reinterpret_cast<char *>(src->d_state) + rows_bytes);
    if (order_enter(src, src->stream)) return -1;
    CK(cudaMemcpyAsync(s_rows, rows.data(), rows_bytes, cudaMemcpyHostToDevice, src->stream));
    records_kernel<false><<<count, 128, 0, src->stream>>>(ts, s_rows, 0, s_rec, words, parts);
    CK(cudaGetLastError());
    // 2. src's order event marks the records ready; dst's stream waits for it (and for dst's own last call)
    if (order_leave(src, src->stream)) return -1;
    CK(cudaSetDevice(dst->device));
    int *d_rows = reinterpret_cast<int *>(dst->d_state);
    float *d_rec = reinterpret_cast<float *>(reinterpret_cast<char *>(dst->d_state) + rows_bytes);
    if (order_enter(dst, dst->stream)) return -1;
    if (dst != src) CK(cudaStreamWaitEvent(dst->stream, src->order_ev, 0));
    // 3. into dst's staging
    if (dst != src) {
        CK(cudaMemcpyAsync(d_rows, rows.data(), rows_bytes, cudaMemcpyHostToDevice, dst->stream));
        if (dst->device != src->device) CK(cudaMemcpyPeerAsync(d_rec, dst->device, s_rec, src->device, bytes - rows_bytes, dst->stream));
        else CK(cudaMemcpyAsync(d_rec, s_rec, bytes - rows_bytes, cudaMemcpyDeviceToDevice, dst->stream));
    }
    // 4. unpack on dst's stream
    records_kernel<true><<<count, 128, 0, dst->stream>>>(td, d_rows + count, 0, d_rec, words, parts);
    CK(cudaGetLastError());
    // 5. both orders end here; the call returns with the copy complete
    if (order_leave(dst, dst->stream)) return -1;
    CK(cudaStreamSynchronize(dst->stream));
    CK(cudaSetDevice(src->device));
    CK(cudaStreamSynchronize(src->stream));

    // host mirrors: frame counters and deferred queues, read from src as it was before the call
    const std::vector<int> sfc = src->fc, sfill = src->dfill;
    const std::vector<float> sq = src->deferred;
    const int sF = src->deferred_fill;
    int q_max = 0;
    for (int k = 0; k < count; k++) q_max = std::max(q_max, sfill[src_rows[k]]);
    const size_t sfr = (size_t)src->n * NB_FEAT, dfr = (size_t)dst->n * NB_FEAT;
    if (q_max > dst->deferred_fill) {       // grow dst's queue at its old end: the other streams read only their last dfill frames
        const int grow = q_max - dst->deferred_fill;
        dst->deferred.resize(dfr * DEFER_MAX);
        float *q = dst->deferred.data();
        memmove(q + dfr * grow, q, sizeof(float) * dfr * dst->deferred_fill);
        std::fill(q, q + dfr * grow, 0.f);
        dst->deferred_fill = q_max;
    }
    const int dF = dst->deferred_fill;
    for (int k = 0; k < count; k++) {
        const int s = src_rows[k], d = dst_rows[k], qn = sfill[s];
        for (int i = 0; i < qn; i++)
            memcpy(dst->deferred.data() + dfr * (dF - qn + i) + (size_t)d * NB_FEAT, sq.data() + sfr * (sF - qn + i) + (size_t)s * NB_FEAT, sizeof(float) * NB_FEAT);
        dst->dfill[d] = qn;
        dst->fc[d] = sfc[s];
    }
    if (!tails) dst->cond_last = -1;
    return 0;
}

// ---- whole-batch snapshot on the device (roll-back after speculative synthesis) ----
// It also holds the frame a tail reads, as the reference's state copy holds gru_a_condition / gru_b_condition / lpc.
struct LPCNetB200Snapshot {
    int n, na, is_float, device;
    StateCopy st;
    std::vector<int> fc; int cond_last; int deferred_fill; std::vector<float> deferred; std::vector<int> dfill;
};
static Fields snapshot_fields(LPCNetB200Snapshot *s) { return state_fields(s->st.ss, s->st.fs, s->st.tail, s->n, s->na, s->is_float); }
void lpcnet_b200_batch_snapshot_destroy(LPCNetB200Snapshot *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    free_state(snapshot_fields(s));
    delete s;
}
LPCNetB200Snapshot *lpcnet_b200_batch_snapshot_create(LPCNetB200Batch *b)
{
    if (!b) { set_error("null batch"); return nullptr; }
    if (cudaSetDevice(b->device) != cudaSuccess) return nullptr;
    LPCNetB200Snapshot *s = new LPCNetB200Snapshot();
    s->n = b->n; s->na = b->model.na; s->is_float = b->model.is_float; s->device = b->device;
    s->fc.assign(b->n, 0); s->dfill.assign(b->n, 0);
    if (!alloc_state(snapshot_fields(s), ALL)) { set_error("snapshot: device allocation failed"); lpcnet_b200_batch_snapshot_destroy(s); return nullptr; }
    return s;
}
static bool snapshot_fits(const LPCNetB200Batch *b, const LPCNetB200Snapshot *s)
{
    if (b && s && s->n == b->n && s->na == b->model.na && s->device == b->device && s->is_float == b->model.is_float) return true;
    set_error("snapshot does not belong to this batch");
    return false;
}
int lpcnet_b200_batch_snapshot_save(LPCNetB200Batch *b, LPCNetB200Snapshot *s)
{
    if (!snapshot_fits(b, s)) return -1;
    CK(cudaSetDevice(b->device));
    if (order_enter(b, b->stream)) return -1;
    if (copy_state(snapshot_fields(s), batch_fields(b, b->cond_last), b->cond_last >= 0 ? ALL : STATE, b->stream)) return -1;
    if (order_leave(b, b->stream)) return -1;
    s->fc = b->fc; s->cond_last = b->cond_last; s->deferred_fill = b->deferred_fill; s->deferred = b->deferred; s->dfill = b->dfill;
    return 0;
}
int lpcnet_b200_batch_snapshot_restore(LPCNetB200Batch *b, const LPCNetB200Snapshot *s)
{
    if (!snapshot_fits(b, s)) return -1;
    CK(cudaSetDevice(b->device));
    if (order_enter(b, b->stream)) return -1;
    const Fields saved = snapshot_fields(const_cast<LPCNetB200Snapshot *>(s));
    if (copy_state(batch_fields(b, TAIL_SLOT), saved, s->cond_last >= 0 ? ALL : STATE, b->stream)) return -1;
    if (order_leave(b, b->stream)) return -1;
    b->fc = s->fc; b->deferred_fill = s->deferred_fill; b->deferred = s->deferred; b->dfill = s->dfill;
    b->cond_last = s->cond_last >= 0 ? TAIL_SLOT : -1;
    return 0;
}

// Test hook: run ONLY the frame-rate kernels on host features for a fresh batch state and return all taps.
// ga [n][nframes][3*na], gb [n][nframes][48], lpc [n][nframes][16] (gamma-weighted, i.e. what the sample loop uses)
int lpcnet_b200_debug_frame_network(LPCNetB200Batch *b, const float *features, int nframes, int feature_stride,
                                                  float *ga, float *gb, float *lpc)
{
    if (!b) { set_error("null batch"); return -1; }
    if (nframes > CHUNK) { set_error("debug_frame_network: at most %d frames", CHUNK); return -1; }
    CK(cudaSetDevice(b->device));
    const int n = b->n, na = b->model.na;
    const size_t fbytes = sizeof(float) * (size_t)n * nframes * feature_stride;
    if (order_sync(b)) return -1;
    if (ensure(b, (void **)&b->d_features, &b->d_features_cap, fbytes)) return -1;
    CK(cudaMemcpyAsync(b->d_features, features, fbytes, cudaMemcpyHostToDevice, b->stream));
    launch_frame_network(b->model, b->fs, b->d_features, (long long)nframes * feature_stride, feature_stride, n, nframes,
                         b->condA, b->condB, b->lpc_raw, b->stream);
    for (int &v : b->fc) v = std::min(1000, v + nframes);
    b->cond_last = nframes - 1;
    const bool isf = b->model.is_float != 0;
    const size_t fA = condA_frame_floats(isf, n, na);
    std::vector<float> hA((size_t)nframes * fA), hB((size_t)nframes * n * 3 * NB), hl((size_t)(nframes + 2) * n * LPC_ORDER), gp(LPC_ORDER);
    CK(cudaMemcpyAsync(hA.data(), b->condA, hA.size() * 4, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaMemcpyAsync(hB.data(), b->condB, hB.size() * 4, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaMemcpyAsync(hl.data(), b->lpc_raw, hl.size() * 4, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaMemcpyAsync(gp.data(), b->model.gamma_pow, LPC_ORDER * 4, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
    const int d = b->model.cfg.end2end ? 0 : b->model.cfg.features_delay;
    for (int s = 0; s < n; s++) for (int f = 0; f < nframes; f++) {
        if (isf) memcpy(ga + ((size_t)s * nframes + f) * 3 * na, &hA[((size_t)f * n + s) * 3 * na], sizeof(float) * 3 * na);
        else for (int g = 0; g < 3; g++) memcpy(ga + ((size_t)s * nframes + f) * 3 * na + (size_t)g * na, &hA[(size_t)f * fA + ((size_t)g * n + s) * (na + 8)], sizeof(float) * na);
        memcpy(gb + ((size_t)s * nframes + f) * 3 * NB, &hB[((size_t)f * n + s) * 3 * NB], sizeof(float) * 3 * NB);
        for (int i = 0; i < LPC_ORDER; i++) lpc[((size_t)s * nframes + f) * LPC_ORDER + i] = hl[((size_t)(f + 2 - d) * n + s) * LPC_ORDER + i] * gp[i];
    }
    return 0;
}

// Test hook (host only, no CUDA): the shared-memory image and its run-time layout words
// layout[8] = {wA, metaA, wB, metaB, image_bytes, total_bytes, nblkA_padded, nblkB_padded}; also returns sm_image in layout[8].
// layout[21] = 1 when the model's accumulator bound allows the conversion-free rounding (DeviceModel::fast_cvt).
int lpcnet_b200_debug_image(const unsigned char *blob, int len, unsigned char *out, size_t cap, uint32_t *layout)
{
    SmemLayout L; Geom G; int fast_cvt = 0;
    int r = debug_build_image(blob, len, out, cap, &L, &G, &fast_cvt);
    if (r < 0) return r;
    layout[0] = L.wA; layout[1] = L.metaA; layout[2] = L.wB; layout[3] = L.metaB; layout[4] = L.image_bytes; layout[5] = L.total_bytes;
    layout[6] = L.nblkA_padded; layout[7] = L.nblkB_padded; layout[8] = L.sm_image;
    layout[9] = G.im_para; layout[10] = G.im_dira; layout[11] = G.im_grpa; layout[12] = G.im_dirb; layout[13] = G.im_wbrec; layout[14] = G.im_parb;
    layout[15] = G.im_fcw; layout[16] = NWC; layout[17] = G.gpw; layout[18] = *reinterpret_cast<const uint32_t *>(out + G.im_fcwn); layout[19] = KPARTS;
    layout[20] = G.na; layout[21] = (uint32_t)fast_cvt;
    return r;
}

// Test hook: the device implementation of the reference's _mm256_rcp_ps (the table in memory) on n host floats.
__global__ void debug_rcp_kernel(const float *x, float *out, int n, const uint16_t *tab16)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = rcp_emul(x[i], tab16);
}
int lpcnet_b200_debug_rcp(LPCNetB200Batch *b, const float *x, float *out, int n)
{
    if (!b || n <= 0) { set_error("debug_rcp: bad arguments"); return -1; }
    CK(cudaSetDevice(b->device));
    float *d = nullptr;
    CK(cudaMalloc(&d, (size_t)2 * n * sizeof(float)));
    CK(cudaMemcpy(d, x, (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
    debug_rcp_kernel<<<(n + 255) / 256, 256, 0, b->stream>>>(d, d + n, n, b->model.rcp16);
    CK(cudaStreamSynchronize(b->stream));
    CK(cudaMemcpy(out, d + n, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    cudaFree(d);
    return 0;
}

// Test hook: the conditioning network's full-range _mm256_rcp_ps and tanh8_approx (devmath.cuh rcp_emul_x86 / tanh_approx_x86)
// on n host floats.
__global__ void debug_tanh_x86_kernel(const float *x, float *out_rcp, float *out_tanh, int n, const uint16_t *tab16)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out_rcp[i] = rcp_emul_x86(x[i], tab16);
    out_tanh[i] = tanh_approx_x86(x[i], tab16);
}
int lpcnet_b200_debug_tanh_x86(LPCNetB200Batch *b, const float *x, float *out_rcp, float *out_tanh, int n)
{
    if (!b || n <= 0) { set_error("debug_tanh_x86: bad arguments"); return -1; }
    CK(cudaSetDevice(b->device));
    float *d = nullptr;
    CK(cudaMalloc(&d, (size_t)3 * n * sizeof(float)));
    CK(cudaMemcpy(d, x, (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
    debug_tanh_x86_kernel<<<(n + 255) / 256, 256, 0, b->stream>>>(d, d + n, d + 2 * n, n, b->model.rcp16);
    CK(cudaStreamSynchronize(b->stream));
    CK(cudaMemcpy(out_rcp, d + n, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(out_tanh, d + 2 * n, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
    cudaFree(d);
    return 0;
}

// Test hook (host only): image of the neuron-per-lane float kernel.  layout = {wA, metaA, wB, metaB, image_bytes, total_bytes,
// nblkA, nblkB, fn_image, fni_neur, fni_dira, fni_para, fni_dirb, fni_parb, fni_wbrec, fni_fcw, dense flag, na}
int lpcnet_b200_debug_image_n(const unsigned char *blob, int len, unsigned char *out, size_t cap, uint32_t *layout)
{
    SmemLayout L; Geom G;
    int r = debug_build_image_n(blob, len, out, cap, &L, &G);
    if (r < 0) return r;
    layout[0] = L.wA; layout[1] = L.metaA; layout[2] = L.wB; layout[3] = L.metaB; layout[4] = L.image_bytes; layout[5] = L.total_bytes;
    layout[6] = L.nblkA_padded; layout[7] = L.nblkB_padded; layout[8] = G.fn_image; layout[9] = G.fni_neur; layout[10] = G.fni_dira; layout[11] = G.fni_para;
    layout[12] = G.fni_dirb; layout[13] = G.fni_parb; layout[14] = G.fni_wbrec; layout[15] = G.fni_fcw; layout[16] = L.wBrecF; layout[17] = G.na;
    return r;
}

// Pinned host memory helpers for callers that want true async H2D/D2H (the benchmark's e2e leg).
void *lpcnet_b200_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { set_error("cudaHostAlloc(%zu) failed", bytes); return nullptr; }
    return p;
}
void lpcnet_b200_host_free(void *p) { if (p) cudaFreeHost(p); }

}  // extern "C"
