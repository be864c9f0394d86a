// multi_api.cu — multi-GPU inside the C-ABI (SURVEY 8e): ONE process, N CUDA devices, no framework on the data path.
//
// Streams never interact (reference: no globals, read-only weights), so a batch of n streams is cut into contiguous
// index ranges, one LPCNetB200Batch per device, weights replicated.  A call enqueues every shard's work on that shard's
// own CUDA stream (H2D features -> frame-rate kernels -> per-sample kernel -> PCM out) and only then waits: the devices run
// concurrently, there is NO collective inside the sample loop.  The one exchange of the path is the PCM gather:
//   * `lpcnet_b200_multi_synthesize` / `_decode` (host in, host out): every device copies its shard's PCM straight into the
//     caller's host buffer over its own PCIe link — no gather step is needed when the consumer is the host;
//   * `..._gather` (host in, PCM gathered in the memory of devices[0]): every finished chunk (<= 16 frames) of a shard is
//     pushed by that device's copy engine over NVLink into the gather buffer (peer access) while the next chunk is being
//     computed (LPCNetB200Batch's PCM sink, batch_api.cu forward_to_sink).
// One process per GPU (torchrun / MPI style) uses the same sink through CUDA IPC instead: lpcnet_b200_ipc_export/_open.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "engine.h"
#include "../../include/lpcnet_b200.h"

using namespace lpcnet_b200;

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_error("%s failed: %s", #call, cudaGetErrorString(e_)); return -1; } } while (0)

struct Shard {
    int device, first, count;
    LPCNetB200Batch *batch;
    cudaStream_t stream;
    void *d_in; size_t d_in_cap;          // features / packets of the shard
    short *d_pcm; size_t d_pcm_cap;
};

struct LPCNetB200Multi {
    int n;
    std::vector<Shard> shards;
    bool peer_ok;                         // every device can write the memory of devices[0]
};

static int grow(void **p, size_t *cap, size_t bytes)
{
    if (*cap >= bytes) return 0;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    CK(cudaMalloc(p, bytes));
    *cap = bytes;
    return 0;
}

extern "C" {

// contiguous shard k of n over `parts`: sizes differ by at most one, earlier shards take the remainder (same rule as
// lpcnet_b200/sharding.py shard_range)
int lpcnet_b200_shard_range(int n, int k, int parts, int *first, int *count)
{
    if (n < 0 || parts <= 0 || k < 0 || k >= parts) { set_error("shard_range: bad arguments"); return -1; }
    const int base = n / parts, rem = n % parts;
    if (first) *first = k * base + std::min(k, rem);
    if (count) *count = base + (k < rem ? 1 : 0);
    return 0;
}

void lpcnet_b200_multi_destroy(LPCNetB200Multi *m)
{
    if (!m) return;
    for (Shard &s : m->shards) {
        cudaSetDevice(s.device);
        if (s.stream) cudaStreamSynchronize(s.stream);
        if (s.batch) lpcnet_b200_batch_destroy(s.batch);
        if (s.d_in) cudaFree(s.d_in);
        if (s.d_pcm) cudaFree(s.d_pcm);
        if (s.stream) cudaStreamDestroy(s.stream);
    }
    delete m;
}

LPCNetB200Multi *lpcnet_b200_multi_create(int n_streams, const unsigned char *blob, int blob_len, const LPCNetB200Config *cfg,
                                          const int *devices, int n_devices)
{
    const int have = lpcnet_b200_device_count();
    if (have <= 0) { set_error("no CUDA device available (this engine has no CPU fallback)"); return nullptr; }
    if (n_devices <= 0 || n_devices > have) { set_error("multi_create: %d devices requested, %d available", n_devices, have); return nullptr; }
    if (n_streams < n_devices) { set_error("multi_create: %d streams cannot be sharded over %d devices", n_streams, n_devices); return nullptr; }
    for (int k = 0; k < n_devices; k++) {
        const int d = devices ? devices[k] : k;
        if (d < 0 || d >= have) { set_error("multi_create: device %d out of range (%d devices)", d, have); return nullptr; }
        for (int j = 0; j < k; j++) if ((devices ? devices[j] : j) == d) { set_error("multi_create: device %d listed twice", d); return nullptr; }
    }
    LPCNetB200Multi *m = new LPCNetB200Multi();
    m->n = n_streams; m->peer_ok = true;
    for (int k = 0; k < n_devices; k++) {
        Shard s; memset(&s, 0, sizeof(s));
        s.device = devices ? devices[k] : k;
        lpcnet_b200_shard_range(n_streams, k, n_devices, &s.first, &s.count);
        m->shards.push_back(s);
    }
    const int dev0 = m->shards[0].device;
    for (Shard &s : m->shards) {
        s.batch = lpcnet_b200_batch_create_ex(s.count, blob, blob_len, cfg, s.device);      // (sets the current device)
        if (!s.batch || cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess) {
            if (s.batch) set_error("multi_create: stream creation failed on device %d", s.device);
            lpcnet_b200_multi_destroy(m); return nullptr;
        }
        if (s.device != dev0) {           // direct NVLink writes into the gather buffer of devices[0]
            int can = 0;
            cudaDeviceCanAccessPeer(&can, s.device, dev0);
            if (can) { cudaError_t e = cudaDeviceEnablePeerAccess(dev0, 0); if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) can = 0; cudaGetLastError(); }
            if (!can) m->peer_ok = false; // copies still work (staged by the driver), only slower
        }
    }
    return m;
}

int lpcnet_b200_multi_streams(const LPCNetB200Multi *m) { return m ? m->n : 0; }
int lpcnet_b200_multi_devices(const LPCNetB200Multi *m) { return m ? (int)m->shards.size() : 0; }
int lpcnet_b200_multi_peer_access(const LPCNetB200Multi *m) { return m && m->peer_ok ? 1 : 0; }

int lpcnet_b200_multi_shard(const LPCNetB200Multi *m, int k, int *device, int *first, int *count)
{
    if (!m || k < 0 || k >= (int)m->shards.size()) { set_error("multi_shard: bad shard index"); return -1; }
    const Shard &s = m->shards[k];
    if (device) *device = s.device;
    if (first) *first = s.first;
    if (count) *count = s.count;
    return 0;
}
// the shard's batch: per-stream lifecycle calls (reset_streams, export/import, snapshots ...) go through it with LOCAL stream ids
LPCNetB200Batch *lpcnet_b200_multi_batch(LPCNetB200Multi *m, int k)
{
    if (!m || k < 0 || k >= (int)m->shards.size()) { set_error("multi_batch: bad shard index"); return nullptr; }
    return m->shards[k].batch;
}

int lpcnet_b200_multi_reset(LPCNetB200Multi *m)
{
    if (!m) { set_error("null multi-batch"); return -1; }
    for (Shard &s : m->shards) if (lpcnet_b200_batch_reset(s.batch)) return -1;
    return 0;
}
int lpcnet_b200_multi_set_codebooks(LPCNetB200Multi *m, const float *cb, size_t n_floats)
{
    if (!m) { set_error("null multi-batch"); return -1; }
    for (Shard &s : m->shards) if (lpcnet_b200_batch_set_codebooks(s.batch, cb, n_floats)) return -1;
    return 0;
}

// Shared body.  in: host features [n][nframes][stride] (packets: [n][npackets][8]); out: host pcm [n][T] (gather_dev == NULL)
// or the gather buffer d_gather [n][T] in the memory of devices[0].
static int run_all(LPCNetB200Multi *m, const void *in, size_t in_row_bytes, int units, int stride, int spf, bool decode,
                   short *pcm_host, short *d_gather)
{
    const long long T = decode ? (long long)units * 640 : (long long)units * spf;
    int rc = 0;
    // enqueue everything on every device first ...
    for (Shard &s : m->shards) {
        CK(cudaSetDevice(s.device));
        const size_t ibytes = in_row_bytes * s.count, pbytes = sizeof(short) * (size_t)T * s.count;
        CK(cudaStreamSynchronize(s.stream));                                   // previous call's users of the staging buffers
        if (grow(&s.d_in, &s.d_in_cap, ibytes) || grow((void **)&s.d_pcm, &s.d_pcm_cap, pbytes)) return -1;
        if (lpcnet_b200_batch_set_pcm_sink(s.batch, d_gather, T, s.first)) return -1;   // NULL removes it
        CK(cudaMemcpyAsync(s.d_in, (const char *)in + in_row_bytes * s.first, ibytes, cudaMemcpyHostToDevice, s.stream));
        const int r = decode ? lpcnet_b200_batch_decode_device(s.batch, (const unsigned char *)s.d_in, units, s.d_pcm, s.stream)
                             : lpcnet_b200_batch_synthesize_device(s.batch, (const float *)s.d_in, units, stride, spf, s.d_pcm, s.stream);
        if (r) { rc = -1; break; }
        if (pcm_host) CK(cudaMemcpyAsync(pcm_host + (size_t)T * s.first, s.d_pcm, pbytes, cudaMemcpyDeviceToHost, s.stream));
    }
    // ... then wait for all of them (also on the error path: nothing may still be reading the caller's buffers)
    for (Shard &s : m->shards) {
        cudaSetDevice(s.device);
        if (cudaStreamSynchronize(s.stream) != cudaSuccess && rc == 0) { set_error("multi: device %d: %s", s.device, cudaGetErrorString(cudaGetLastError())); rc = -1; }
    }
    return rc;
}

int lpcnet_b200_multi_synthesize(LPCNetB200Multi *m, const float *features, int nframes, int feature_stride, int samples_per_frame, short *pcm)
{
    if (!m || !features || !pcm) { set_error("multi_synthesize: null argument"); return -1; }
    if (nframes <= 0) return 0;
    return run_all(m, features, sizeof(float) * (size_t)nframes * feature_stride, nframes, feature_stride, samples_per_frame, false, pcm, nullptr);
}
int lpcnet_b200_multi_synthesize_gather(LPCNetB200Multi *m, const float *features, int nframes, int feature_stride, int samples_per_frame, short *d_pcm)
{
    if (!m || !features || !d_pcm) { set_error("multi_synthesize_gather: null argument"); return -1; }
    if (nframes <= 0) return 0;
    return run_all(m, features, sizeof(float) * (size_t)nframes * feature_stride, nframes, feature_stride, samples_per_frame, false, nullptr, d_pcm);
}
int lpcnet_b200_multi_decode(LPCNetB200Multi *m, const unsigned char *packets, int npackets, short *pcm)
{
    if (!m || !packets || !pcm) { set_error("multi_decode: null argument"); return -1; }
    if (npackets <= 0) return 0;
    return run_all(m, packets, (size_t)npackets * 8, npackets, 0, FRAME_SIZE, true, pcm, nullptr);
}
int lpcnet_b200_multi_decode_gather(LPCNetB200Multi *m, const unsigned char *packets, int npackets, short *d_pcm)
{
    if (!m || !packets || !d_pcm) { set_error("multi_decode_gather: null argument"); return -1; }
    if (npackets <= 0) return 0;
    return run_all(m, packets, (size_t)npackets * 8, npackets, 0, FRAME_SIZE, true, nullptr, d_pcm);
}

// memory on a given device (the gather buffer lives on devices[0])
void *lpcnet_b200_device_alloc_on(int device, size_t bytes)
{
    int cur = 0;
    cudaGetDevice(&cur);
    void *p = nullptr;
    if (cudaSetDevice(device) != cudaSuccess || cudaMalloc(&p, bytes) != cudaSuccess) { set_error("device_alloc_on(%d, %zu) failed: %s", device, bytes, cudaGetErrorString(cudaGetLastError())); p = nullptr; }
    cudaSetDevice(cur);
    return p;
}

}  // extern "C"
