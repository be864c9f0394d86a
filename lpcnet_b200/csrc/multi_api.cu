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
// Multi-GPU groups (lpcnet_b200_multi_group_*) serve several models, one LPCNetB200Multi each over the same devices, the same way:
// per device one group over the members' shards, and the gather forwarded from inside the group's chunk loop
// (batch_api.cu group_call with forward targets) instead of through the shard batches' sinks.
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
static int run_all(LPCNetB200Multi *m, const CallShape &c, const void *in, short *pcm_host, short *d_gather)
{
    const long long T = c.pcm_samples();
    int rc = 0;
    // enqueue everything on every device first ...
    for (Shard &s : m->shards) {
        CK(cudaSetDevice(s.device));
        const size_t ibytes = c.in_bytes() * s.count, pbytes = sizeof(short) * (size_t)T * s.count;
        CK(cudaStreamSynchronize(s.stream));                                   // previous call's users of the staging buffers
        if (grow_buffer(&s.d_in, &s.d_in_cap, ibytes) || grow_buffer((void **)&s.d_pcm, &s.d_pcm_cap, pbytes)) return -1;
        if (lpcnet_b200_batch_set_pcm_sink(s.batch, d_gather, T, s.first)) return -1;   // NULL removes it
        CK(cudaMemcpyAsync(s.d_in, (const char *)in + c.in_bytes() * s.first, ibytes, cudaMemcpyHostToDevice, s.stream));
        const int r = c.decode ? lpcnet_b200_batch_decode_device(s.batch, (const unsigned char *)s.d_in, c.units, s.d_pcm, s.stream)
                               : lpcnet_b200_batch_synthesize_device(s.batch, (const float *)s.d_in, c.units, c.stride, c.spf, s.d_pcm, s.stream);
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
    return run_all(m, CallShape::synthesis(nframes, feature_stride, samples_per_frame), features, pcm, nullptr);
}
int lpcnet_b200_multi_synthesize_gather(LPCNetB200Multi *m, const float *features, int nframes, int feature_stride, int samples_per_frame, short *d_pcm)
{
    if (!m || !features || !d_pcm) { set_error("multi_synthesize_gather: null argument"); return -1; }
    if (nframes <= 0) return 0;
    return run_all(m, CallShape::synthesis(nframes, feature_stride, samples_per_frame), features, nullptr, d_pcm);
}
int lpcnet_b200_multi_decode(LPCNetB200Multi *m, const unsigned char *packets, int npackets, short *pcm)
{
    if (!m || !packets || !pcm) { set_error("multi_decode: null argument"); return -1; }
    if (npackets <= 0) return 0;
    return run_all(m, CallShape::packets(npackets), packets, pcm, nullptr);
}
int lpcnet_b200_multi_decode_gather(LPCNetB200Multi *m, const unsigned char *packets, int npackets, short *d_pcm)
{
    if (!m || !packets || !d_pcm) { set_error("multi_decode_gather: null argument"); return -1; }
    if (npackets <= 0) return 0;
    return run_all(m, CallShape::packets(npackets), packets, nullptr, d_pcm);
}

// ---- multi-GPU groups: several models, each an LPCNetB200Multi over the same devices, in one call ----
// Device k runs one LPCNetB200Group over shard k of every member.  Job rows are member 0's streams, then member 1's, ...; on device k
// the rows of member m are base[m] + first_mk .. + count_mk, staged in the device's buffers as one block per member, in member order
// (the group's own row layout).
struct MGDevice {
    int device, rows;                     // rows: sum over the members of their shard's streams on this device
    LPCNetB200Group *group;
    cudaStream_t stream;
    void *d_in; size_t d_in_cap;
    short *d_pcm; size_t d_pcm_cap;
};

struct LPCNetB200MultiGroup {
    int n;
    std::vector<LPCNetB200Multi *> m;
    std::vector<int> base;                // first job row of each member
    std::vector<MGDevice> dev;
};

void lpcnet_b200_multi_group_destroy(LPCNetB200MultiGroup *mg)
{
    if (!mg) return;
    for (MGDevice &d : mg->dev) {
        cudaSetDevice(d.device);
        if (d.stream) cudaStreamSynchronize(d.stream);
        if (d.group) lpcnet_b200_group_destroy(d.group);
        if (d.d_in) cudaFree(d.d_in);
        if (d.d_pcm) cudaFree(d.d_pcm);
        if (d.stream) cudaStreamDestroy(d.stream);
    }
    delete mg;
}

LPCNetB200MultiGroup *lpcnet_b200_multi_group_create(LPCNetB200Multi *const *members, int count)
{
    if (!members || count < 1 || count > GROUP_MAX) { set_error("multi_group_create: 1..%d member multis", GROUP_MAX); return nullptr; }
    int na0 = 0;
    for (int k = 0; k < count; k++) {
        const LPCNetB200Multi *m = members[k];
        if (!m) { set_error("multi_group_create: member %d is NULL", k); return nullptr; }
        for (int j = 0; j < k; j++) if (members[j] == m) { set_error("multi_group_create: member %d is listed twice (also member %d)", k, j); return nullptr; }
        const std::vector<Shard> &s = m->shards, &s0 = members[0]->shards;
        bool same = s.size() == s0.size();
        for (size_t i = 0; same && i < s.size(); i++) same = s[i].device == s0[i].device;
        if (!same) { set_error("multi_group_create: member %d runs on other devices than member 0 (the device lists must be equal, in order)", k); return nullptr; }
        int na = 0;
        lpcnet_b200_batch_model_info(s[0].batch, &na, nullptr);
        if (k == 0) na0 = na;
        if (na != na0) { set_error("multi_group_create: member %d has %d GRU_A units, member 0 has %d", k, na, na0); return nullptr; }
        const int fl = lpcnet_b200_batch_is_float(s[0].batch), fl0 = lpcnet_b200_batch_is_float(s0[0].batch);
        if (fl != fl0) {
            set_error("multi_group_create: member %d holds %s model, member 0 %s one; the members are all int8 or all float", k,
                      fl ? "a float" : "an int8", fl0 ? "a float" : "an int8");
            return nullptr;
        }
    }
    LPCNetB200MultiGroup *mg = new LPCNetB200MultiGroup();
    mg->m.assign(members, members + count);
    for (LPCNetB200Multi *m : mg->m) { mg->base.push_back(mg->n); mg->n += m->n; }
    const size_t nd = members[0]->shards.size();
    for (size_t k = 0; k < nd; k++) {
        MGDevice d; memset(&d, 0, sizeof(d));
        d.device = members[0]->shards[k].device;
        mg->dev.push_back(d);
    }
    for (size_t k = 0; k < nd; k++) {
        MGDevice &d = mg->dev[k];
        LPCNetB200Batch *b[GROUP_MAX];
        for (int j = 0; j < count; j++) { b[j] = members[j]->shards[k].batch; d.rows += members[j]->shards[k].count; }
        d.group = lpcnet_b200_group_create(b, count);          // (sets the current device)
        if (!d.group || cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking) != cudaSuccess) {
            if (d.group) set_error("multi_group_create: stream creation failed on device %d", d.device);
            lpcnet_b200_multi_group_destroy(mg); return nullptr;
        }
    }
    return mg;
}

int lpcnet_b200_multi_group_streams(const LPCNetB200MultiGroup *mg) { return mg ? mg->n : 0; }
LPCNetB200Group *lpcnet_b200_multi_group_group(LPCNetB200MultiGroup *mg, int k)
{
    if (!mg || k < 0 || k >= (int)mg->dev.size()) { set_error("multi_group_group: bad device index"); return nullptr; }
    return mg->dev[k].group;
}

// One device's share of a checked call, enqueued on its stream: every member's rows up, then the group call, which forwards each
// chunk to the gather buffer if there is one
static int mg_enqueue(LPCNetB200MultiGroup *mg, size_t k, const CallShape &c, const void *in, short *d_gather)
{
    MGDevice &d = mg->dev[k];
    const long long T = c.pcm_samples();
    CK(cudaSetDevice(d.device));
    if (grow_buffer(&d.d_in, &d.d_in_cap, c.in_bytes() * d.rows) || grow_buffer((void **)&d.d_pcm, &d.d_pcm_cap, sizeof(short) * (size_t)T * d.rows)) return -1;
    PcmTarget fwd[GROUP_MAX];
    int local = 0;
    for (size_t j = 0; j < mg->m.size(); j++) {
        const Shard &s = mg->m[j]->shards[k];
        const long long row = mg->base[j] + s.first;
        fwd[j] = PcmTarget{d_gather, T, row};
        CK(cudaMemcpyAsync((char *)d.d_in + c.in_bytes() * local, (const char *)in + c.in_bytes() * row, c.in_bytes() * s.count, cudaMemcpyHostToDevice, d.stream));
        local += s.count;
    }
    const void *pin[GROUP_MAX]; short *pcm[GROUP_MAX];
    group_rows(d.group, c, d.d_in, d.d_pcm, nullptr, pin, pcm);
    return group_call(d.group, c, pin, pcm, d_gather ? fwd : nullptr, d.stream);
}
// ... and its rows of every member down to the host
static int mg_download(LPCNetB200MultiGroup *mg, size_t k, long long T, short *pcm_host)
{
    MGDevice &d = mg->dev[k];
    CK(cudaSetDevice(d.device));
    int local = 0;
    for (size_t j = 0; j < mg->m.size(); j++) {
        const Shard &s = mg->m[j]->shards[k];
        CK(cudaMemcpyAsync(pcm_host + (size_t)T * (mg->base[j] + s.first), d.d_pcm + (size_t)T * local, sizeof(short) * (size_t)T * s.count,
                           cudaMemcpyDeviceToHost, d.stream));
        local += s.count;
    }
    return 0;
}

static int mg_run(LPCNetB200MultiGroup *mg, const CallShape &c, const void *in, short *pcm_host, short *d_gather)
{
    for (MGDevice &d : mg->dev)          // refuse before anything is enqueued on any device
        if (group_check(d.group, c, false)) return -1;
    int rc = 0;
    // enqueue the work of every device first, the copies to the host after it (a copy to pageable memory returns only once it
    // is done: it must not hold back the next device's work) ...
    for (size_t k = 0; k < mg->dev.size() && rc == 0; k++) rc = mg_enqueue(mg, k, c, in, d_gather);
    for (size_t k = 0; pcm_host && k < mg->dev.size() && rc == 0; k++) rc = mg_download(mg, k, c.pcm_samples(), pcm_host);
    // ... then wait for all of them (also on the error path: nothing may still be reading the caller's buffers)
    for (MGDevice &d : mg->dev) {
        cudaSetDevice(d.device);
        if (cudaStreamSynchronize(d.stream) != cudaSuccess && rc == 0) { set_error("multi_group: device %d: %s", d.device, cudaGetErrorString(cudaGetLastError())); rc = -1; }
    }
    return rc;
}

int lpcnet_b200_multi_group_synthesize(LPCNetB200MultiGroup *mg, const float *features, int nframes, int feature_stride, int samples_per_frame, short *pcm)
{
    if (!mg || !features || !pcm) { set_error("multi_group_synthesize: null argument"); return -1; }
    if (nframes <= 0) return 0;
    return mg_run(mg, CallShape::synthesis(nframes, feature_stride, samples_per_frame), features, pcm, nullptr);
}
int lpcnet_b200_multi_group_synthesize_gather(LPCNetB200MultiGroup *mg, const float *features, int nframes, int feature_stride, int samples_per_frame, short *d_pcm)
{
    if (!mg || !features || !d_pcm) { set_error("multi_group_synthesize_gather: null argument"); return -1; }
    if (nframes <= 0) return 0;
    return mg_run(mg, CallShape::synthesis(nframes, feature_stride, samples_per_frame), features, nullptr, d_pcm);
}
int lpcnet_b200_multi_group_decode(LPCNetB200MultiGroup *mg, const unsigned char *packets, int npackets, short *pcm)
{
    if (!mg || !packets || !pcm) { set_error("multi_group_decode: null argument"); return -1; }
    if (npackets <= 0) return 0;
    return mg_run(mg, CallShape::packets(npackets), packets, pcm, nullptr);
}
int lpcnet_b200_multi_group_decode_gather(LPCNetB200MultiGroup *mg, const unsigned char *packets, int npackets, short *d_pcm)
{
    if (!mg || !packets || !d_pcm) { set_error("multi_group_decode_gather: null argument"); return -1; }
    if (npackets <= 0) return 0;
    return mg_run(mg, CallShape::packets(npackets), packets, nullptr, d_pcm);
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
