// mixed_api.cu — mixed groups (lpcnet_b200_mixed_group_*): batches of different GRU_A sizes and flavours on one device in one call.
//
// The per-sample kernels are compiled once per GRU_A size, and the int8 and float kernels differ in warp roles, registers and
// shared memory, so one launch cannot hold two shapes.  A mixed group holds one ordinary group per (GRU_A size, flavour) class,
// all planned with ONE streams-per-CTA value chosen so that the CTAs of all classes together fit on the SMs (batch_api.cu
// mixed_plan), and runs the classes' group calls on different CUDA streams.  A CTA of these kernels never waits on another CTA,
// so the classes' launches can all be resident at once and the call costs about the slowest class instead of the sum.  Whether
// the hardware overlaps them is its choice; the results never depend on it.
#include <cstdlib>
#include <cstring>
#include "engine.h"
#include "../../include/lpcnet_b200.h"

using namespace lpcnet_b200;

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_error("%s failed: %s", #call, cudaGetErrorString(e_)); return -1; } } while (0)

struct LPCNetB200MixedGroup {
    int device, n_total, classes;
    LPCNetB200Group *g[GROUP_MAX];              // class c's group
    int members[GROUP_MAX];                     // class c's member count
    int rows[GROUP_MAX][GROUP_MAX];             // rows[c][j]: first mixed-group row of member j of class c
    cudaStream_t stream[GROUP_MAX];             // [0]: host-pointer calls; [c > 0]: class c's share of every call
    cudaEvent_t fork, done, join[GROUP_MAX];    // fork .. done: the last call on its stream (last_call_ms)
    bool timed;
    void *d_in; size_t d_in_cap;                // staging of the host-pointer calls
    short *d_pcm; size_t d_pcm_cap;
};

extern "C" {

void lpcnet_b200_mixed_group_destroy(LPCNetB200MixedGroup *mg)
{
    if (!mg) return;
    cudaSetDevice(mg->device);
    for (int c = 0; c < mg->classes; c++) {
        if (mg->stream[c]) { cudaStreamSynchronize(mg->stream[c]); cudaStreamDestroy(mg->stream[c]); }
        if (mg->join[c]) cudaEventDestroy(mg->join[c]);
        if (mg->g[c]) lpcnet_b200_group_destroy(mg->g[c]);
    }
    if (mg->fork) cudaEventDestroy(mg->fork);
    if (mg->done) cudaEventDestroy(mg->done);
    if (mg->d_in) cudaFree(mg->d_in);
    if (mg->d_pcm) cudaFree(mg->d_pcm);
    delete mg;
}

LPCNetB200MixedGroup *lpcnet_b200_mixed_group_create(LPCNetB200Batch *const *batches, int count)
{
    if (group_members_check(batches, count, "mixed_group_create", false)) return nullptr;
    int n[GROUP_MAX], na[GROUP_MAX], fl[GROUP_MAX];
    for (int k = 0; k < count; k++) {
        n[k] = lpcnet_b200_batch_streams(batches[k]);
        lpcnet_b200_batch_model_info(batches[k], &na[k], nullptr);
        fl[k] = lpcnet_b200_batch_is_float(batches[k]);
    }
    const int device = batch_device(batches[0]);
    if (cudaSetDevice(device) != cudaSuccess) { set_error("mixed_group_create: cudaSetDevice(%d) failed", device); return nullptr; }
    const char *e = getenv("LPCNET_B200_STREAMS_PER_CTA");
    int spc, class_of[GROUP_MAX], class_ctas[GROUP_MAX];
    bool class_neuron[GROUP_MAX];
    const int classes = mixed_plan(n, na, fl, count, device_sms(device), e ? atoi(e) : 0, getenv("LPCNET_B200_FLOAT_LANE_STREAM") != nullptr,
                                   &spc, class_of, class_ctas, class_neuron);
    LPCNetB200MixedGroup *mg = new LPCNetB200MixedGroup();
    mg->device = device; mg->classes = classes;
    LPCNetB200Batch *cb[GROUP_MAX][GROUP_MAX];
    for (int k = 0; k < count; k++) {
        const int c = class_of[k];
        cb[c][mg->members[c]] = batches[k];
        mg->rows[c][mg->members[c]++] = mg->n_total;
        mg->n_total += n[k];
    }
    bool ok = cudaEventCreate(&mg->fork) == cudaSuccess && cudaEventCreate(&mg->done) == cudaSuccess;
    for (int c = 0; ok && c < classes; c++) {
        mg->g[c] = group_init(cb[c], mg->members[c], spc);
        if (!mg->g[c]) { lpcnet_b200_mixed_group_destroy(mg); return nullptr; }
        ok = cudaStreamCreateWithFlags(&mg->stream[c], cudaStreamNonBlocking) == cudaSuccess &&
             cudaEventCreateWithFlags(&mg->join[c], cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) { set_error("mixed_group_create: stream / event creation failed"); lpcnet_b200_mixed_group_destroy(mg); return nullptr; }
    return mg;
}

int lpcnet_b200_mixed_group_streams(const LPCNetB200MixedGroup *mg) { return mg ? mg->n_total : 0; }
int lpcnet_b200_mixed_group_classes(const LPCNetB200MixedGroup *mg) { return mg ? mg->classes : 0; }
LPCNetB200Group *lpcnet_b200_mixed_group_group(LPCNetB200MixedGroup *mg, int c)
{
    if (!mg || c < 0 || c >= mg->classes) { set_error("mixed_group_group: bad class index"); return nullptr; }
    return mg->g[c];
}

}  // extern "C"

// What a call refuses, in the order of a group call: a member with a PCM sink, NULL buffers, then what any class's group call of
// shape c would refuse.  Returns 1 for a call without units: nothing to do.
static int mx_check(LPCNetB200MixedGroup *mg, const CallShape &c, const void *in, const void *out)
{
    if (!mg) { set_error("null mixed group"); return -1; }
    for (int k = 0; k < mg->classes; k++) if (group_check(mg->g[k], CallShape{}, true)) return -1;
    CK(cudaSetDevice(mg->device));
    if (c.units <= 0) return 1;
    if (!in || !out) { set_error("null buffer"); return -1; }
    for (int k = 0; k < mg->classes; k++) if (group_check(mg->g[k], c, false)) return -1;
    return 0;
}

// One checked call on device buffers `in` (features or packets, [sum n] rows) and `d_pcm`, its completion on `st`: class 0 on st,
// class k > 0 on stream[k] after the fork, every class stream joined back into st (also after an error, so that nothing the call
// enqueued outlives it on st)
static int mx_run(LPCNetB200MixedGroup *mg, const CallShape &c, const void *in, short *d_pcm, cudaStream_t st)
{
    CK(cudaEventRecord(mg->fork, st));
    int rc = 0, started = 0;
    for (int k = 0; k < mg->classes && rc == 0; k++) {
        cudaStream_t cs = k ? mg->stream[k] : st;
        if (k && cudaStreamWaitEvent(cs, mg->fork, 0) != cudaSuccess) { set_error("mixed_group: fork failed"); rc = -1; break; }
        started++;
        const void *pin[GROUP_MAX]; short *pcm[GROUP_MAX];
        group_rows(mg->g[k], c, in, d_pcm, mg->rows[k], pin, pcm);
        rc = group_call(mg->g[k], c, pin, pcm, nullptr, cs);
    }
    for (int k = 1; k < started; k++) {
        CK(cudaEventRecord(mg->join[k], mg->stream[k]));
        CK(cudaStreamWaitEvent(st, mg->join[k], 0));
    }
    CK(cudaEventRecord(mg->done, st));
    mg->timed = true;
    return rc;
}

static int mx_device(LPCNetB200MixedGroup *mg, const CallShape &c, const void *d_in, short *d_pcm, void *cuda_stream)
{
    const int r = mx_check(mg, c, d_in, d_pcm);
    if (r) return r < 0 ? -1 : 0;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : mg->stream[0];
    if (mx_run(mg, c, d_in, d_pcm, st)) return -1;
    if (!cuda_stream) CK(cudaStreamSynchronize(st));
    return 0;
}

// host-pointer calls: the rows go through the mixed group's own staging buffers on stream[0]; returns once the PCM is on the host
static int mx_host(LPCNetB200MixedGroup *mg, const CallShape &c, const void *in, short *pcm)
{
    const int r = mx_check(mg, c, in, pcm);
    if (r) return r < 0 ? -1 : 0;
    const size_t in_bytes = c.in_bytes() * mg->n_total, pcm_bytes = sizeof(short) * c.pcm_samples() * mg->n_total;
    cudaStream_t st = mg->stream[0];
    // (earlier host calls are complete and `_device` calls never touch these buffers: nothing can still be using them)
    if (grow_buffer(&mg->d_in, &mg->d_in_cap, in_bytes) || grow_buffer((void **)&mg->d_pcm, &mg->d_pcm_cap, pcm_bytes)) return -1;
    CK(cudaMemcpyAsync(mg->d_in, in, in_bytes, cudaMemcpyHostToDevice, st));
    int rc = mx_run(mg, c, mg->d_in, mg->d_pcm, st);
    if (rc == 0) CK(cudaMemcpyAsync(pcm, mg->d_pcm, pcm_bytes, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return rc;
}

extern "C" {

int lpcnet_b200_mixed_group_synthesize(LPCNetB200MixedGroup *mg, const float *features, int nframes, int feature_stride,
                                       int samples_per_frame, short *pcm)
{
    return mx_host(mg, CallShape::synthesis(nframes, feature_stride, samples_per_frame), features, pcm);
}

int lpcnet_b200_mixed_group_synthesize_device(LPCNetB200MixedGroup *mg, const float *d_features, int nframes, int feature_stride,
                                              int samples_per_frame, short *d_pcm, void *cuda_stream)
{
    return mx_device(mg, CallShape::synthesis(nframes, feature_stride, samples_per_frame), d_features, d_pcm, cuda_stream);
}

int lpcnet_b200_mixed_group_decode(LPCNetB200MixedGroup *mg, const unsigned char *packets, int npackets, short *pcm)
{
    return mx_host(mg, CallShape::packets(npackets), packets, pcm);
}

int lpcnet_b200_mixed_group_decode_device(LPCNetB200MixedGroup *mg, const unsigned char *d_packets, int npackets, short *d_pcm,
                                          void *cuda_stream)
{
    return mx_device(mg, CallShape::packets(npackets), d_packets, d_pcm, cuda_stream);
}

float lpcnet_b200_mixed_group_last_call_ms(const LPCNetB200MixedGroup *mg)
{
    if (!mg) return -1.f;
    if (!mg->timed) return 0.f;
    float ms = 0.f;
    if (cudaSetDevice(mg->device) != cudaSuccess || cudaEventSynchronize(mg->done) != cudaSuccess ||
        cudaEventElapsedTime(&ms, mg->fork, mg->done) != cudaSuccess) return -1.f;
    return ms;
}

}  // extern "C"
