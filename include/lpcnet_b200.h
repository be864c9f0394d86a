/* lpcnet_b200.h — batched C-ABI of the H100-native LPCNet synthesis engine (the throughput surface).
 *
 * The reference API (include/lpcnet.h) drives ONE stream, 160 samples per call.  The hot path
 * (reference src/lpcnet.c:235-271 `lpcnet_synthesize_tail_impl` -> :146 `run_sample_network`) is strictly serial
 * inside a stream, so GPU throughput comes from stepping thousands of independent streams in lockstep.  This
 * header is the extension SURVEY.md 8(b) calls for: the same operations as `lpcnet_synthesize` /
 * `lpcnet_decode`, applied to a batch of independent streams that all start from a fresh `lpcnet_create()` state
 * (reference src/lpcnet.c:174-200: zero state, RNG seeded with "LPCNet").
 *
 * Plain C: pointers + sizes only.  Host-pointer entry points copy features in and PCM out inside the call;
 * `_device` variants take CUDA device pointers (already resident inputs) and a CUDA stream handle.
 * All functions return 0 on success, negative on error (message: lpcnet_b200_last_error()).
 */
#ifndef LPCNET_B200_H
#define LPCNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifndef LPCNET_EXPORT
# if defined(__GNUC__)
#  define LPCNET_EXPORT __attribute__ ((visibility ("default")))
# else
#  define LPCNET_EXPORT
# endif
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct LPCNetB200Batch LPCNetB200Batch;
typedef struct LPCNetB200Snapshot LPCNetB200Snapshot;

/* The three per-model switches the reference bakes into the generated nnet_data.h (training_tf2/dump_lpcnet.py:306-329)
 * instead of the weight blob.  A negative / non-positive field means "take it from the blob's `lpcnet_b200_config`
 * metadata record (written by lpcnet_b200_write_blob / tools/import_nnet_data.py) or, failing that, the reference default". */
typedef struct LPCNetB200Config {
    float lpc_gamma;        /* LPC_GAMMA: lpc_weighting factor (src/freq.c:299-308); default 1 (none) */
    int features_delay;     /* FEATURES_DELAY 0..2: look-ahead frames (src/lpcnet.c:101,109-115,239); default 2 */
    int end2end;            /* END2END: LPC from the network's reflection coefficients (src/lpcnet.c:57-78,107-108); default 0 */
} LPCNetB200Config;

/* One named array of a model blob: the reference's WeightArray (src/nnet.h:43-48).  type: 0 float, 1 int, 2 qweight (int8);
 * size in bytes. */
typedef struct LPCNetB200Array {
    const char *name;
    int type;
    int size;
    const void *data;
} LPCNetB200Array;

/* == model blob I/O (host only, no CUDA) ==
 * lpcnet_b200_write_blob: serialise arrays to the "DNNw" weight-blob format exactly like the reference's write_weights()
 * (src/write_lpcnet_weights.c:47-67: 64-byte WeightHead, payload zero-padded to a multiple of 64 bytes).  With cfg != NULL the
 * three switches the reference leaves in nnet_data.h travel as one extra record `lpcnet_b200_config` (float[4]: LPC_GAMMA,
 * FEATURES_DELAY, END2END, format version) which the reference's own loader ignores.  out == NULL: returns the size needed.
 * Returns the number of bytes written, < 0 on error. */
LPCNET_EXPORT long long lpcnet_b200_write_blob(const LPCNetB200Array *arrays, int count, const LPCNetB200Config *cfg,
                                               unsigned char *out, size_t cap);
LPCNET_EXPORT int lpcnet_b200_write_blob_file(const char *path, const LPCNetB200Array *arrays, int count, const LPCNetB200Config *cfg);
/* parse_weights() (src/parse_lpcnet_weights.c:37-76): lists the records of a blob (entries point into `blob`).  Returns the
 * number of records (may exceed cap; only cap are filled), < 0 if the blob is malformed. */
LPCNET_EXPORT int lpcnet_b200_parse_blob(const unsigned char *blob, int len, LPCNetB200Array *arrays, int cap);
/* The blob's `lpcnet_b200_config` record: 1 = found (cfg filled), 0 = the blob has none, < 0 malformed blob. */
LPCNET_EXPORT int lpcnet_b200_blob_config(const unsigned char *blob, int len, LPCNetB200Config *cfg);
/* Whole-file read (weights_blob.bin, .f32 feature files, packet files): out == NULL returns the size. */
LPCNET_EXPORT long long lpcnet_b200_read_file(const char *path, unsigned char *out, size_t cap);

/* Number of usable CUDA devices (0 => the engine cannot run; there is no CPU fallback). */
LPCNET_EXPORT int lpcnet_b200_device_count(void);
/* Last error message of the calling thread ("" if none). */
LPCNET_EXPORT const char *lpcnet_b200_last_error(void);
/* Library/ABI version: major*10000 + minor*100 + patch. */
LPCNET_EXPORT int lpcnet_b200_version(void);

/* Create `n_streams` independent synthesis streams on CUDA device `device`, all using the model in the "DNNw"
 * blob (same format/validation as reference lpcnet_load_model, src/lpcnet.c:202 + src/parse_lpcnet_weights.c:115-221;
 * both the int8 DOT_PROD and the float flavour are accepted and select the arithmetic).  `lpc_gamma` is the
 * reference's compile-time LPC_GAMMA (generated nnet_data.h; training_tf2/dump_lpcnet.py:313-319); pass 1.0f for
 * "no weighting".  Returns NULL on error. */
LPCNET_EXPORT LPCNetB200Batch *lpcnet_b200_batch_create(int n_streams, const unsigned char *blob, int blob_len,
                                                        float lpc_gamma, int device);
/* Same with the per-model switches given explicitly (NULL: blob metadata / defaults).  The number of GRU_A units is read
 * from the blob (128, 256 or 384: training_tf2/train_lpcnet.py --grua-size); GRU_B = 16 and cond = 128 are fixed. */
LPCNET_EXPORT LPCNetB200Batch *lpcnet_b200_batch_create_ex(int n_streams, const unsigned char *blob, int blob_len,
                                                           const LPCNetB200Config *cfg, int device);
LPCNET_EXPORT void lpcnet_b200_batch_destroy(LPCNetB200Batch *b);
/* GRU_A units and the switches in effect. */
LPCNET_EXPORT int lpcnet_b200_batch_model_info(const LPCNetB200Batch *b, int *gru_a_units, LPCNetB200Config *cfg);
/* lpcnet_reset() (reference src/lpcnet.c:174) applied to every stream.  It also clears the decoder memory (the previous
 * superframe's cepstrum, LPCNetDecState.vq_mem), as lpcnet_decoder_init() does to a loaded state: a reset stream starts a new
 * utterance. */
LPCNET_EXPORT int lpcnet_b200_batch_reset(LPCNetB200Batch *b);
/* lpcnet_reset() for the listed streams only: they start a new utterance (two silent frames, fresh RNG, decoder memory
 * cleared as above) while the other streams of the batch carry on.  Every stream has its own frame counter. */
LPCNET_EXPORT int lpcnet_b200_batch_reset_streams(LPCNetB200Batch *b, const int *streams, int count);
/* lpcnet_reset_signal() (reference src/lpcnet.c:226-233, used by the PLC): clears the sample-rate state only; the 100 Hz state
 * and the decoder memory stay. */
LPCNET_EXPORT int lpcnet_b200_batch_reset_signal(LPCNetB200Batch *b);
LPCNET_EXPORT int lpcnet_b200_batch_streams(const LPCNetB200Batch *b);

/* VQ codebooks for the decoder front-end (reference src/lpcnet_dec.c:129-143 reads ceps_codebook1..3 [1024][17]
 * and ceps_codebook_diff4 [4096][18]; the reference links them from the un-shipped ceps_codebooks.c).
 * `cb` = the four arrays concatenated in that order (3*1024*17 + 4096*18 floats). */
LPCNET_EXPORT int lpcnet_b200_batch_set_codebooks(LPCNetB200Batch *b, const float *cb, size_t n_floats);

/* == lpcnet_synthesize() per stream, `nframes` times ==
 * features: [n_streams][nframes][feature_stride] floats (first 20 of each frame used; stride 20 or 36 typical)
 * pcm     : [n_streams][nframes*samples_per_frame] int16
 * samples_per_frame is the reference's N argument (160 in the demo/decoder; any N >= 1 like the reference). */
LPCNET_EXPORT int lpcnet_b200_batch_synthesize(LPCNetB200Batch *b, const float *features, int nframes,
                                               int feature_stride, int samples_per_frame, short *pcm);
LPCNET_EXPORT int lpcnet_b200_batch_synthesize_device(LPCNetB200Batch *b, const float *d_features, int nframes,
                                                      int feature_stride, int samples_per_frame, short *d_pcm,
                                                      void *cuda_stream);

/* == lpcnet_synthesize_impl(st, features, out, N, preload) (reference src/lpcnet.c:273-277; PLC entry point) ==
 * The first `preload` samples of the call's FIRST frame are teacher-forced: the network runs (state and RNG advance) but the
 * excitation is derived from the signal the caller supplies in pcm[s][0..preload) and those samples are not overwritten
 * (src/lpcnet.c:256-259,269). */
LPCNET_EXPORT int lpcnet_b200_batch_synthesize_ex(LPCNetB200Batch *b, const float *features, int nframes,
                                                  int feature_stride, int samples_per_frame, short *pcm, int preload);
LPCNET_EXPORT int lpcnet_b200_batch_synthesize_device_ex(LPCNetB200Batch *b, const float *d_features, int nframes,
                                                         int feature_stride, int samples_per_frame, short *d_pcm,
                                                         int preload, void *cuda_stream);
/* == the other internal entry points the reference's PLC uses (src/lpcnet_private.h:125-133), batched ==
 * run_frame_network (src/lpcnet.c:82-120) only: advances the 100 Hz state, keeps the last frame's conditioning */
LPCNET_EXPORT int lpcnet_b200_batch_run_frame_network(LPCNetB200Batch *b, const float *features, int nframes, int feature_stride);
/* lpcnet_synthesize_tail_impl (src/lpcnet.c:235-271): `samples` samples with the conditioning and LPC of the last
 * _synthesize* or _run_frame_network call; pcm [n_streams][samples].  As in the reference, what the tail reads is per-stream
 * state: a flush leaves it as it was; a reset zeroes it for the streams it resets (so a tail right after one gives zeros);
 * a snapshot restore brings back what the snapshot saved.  After an _import_state the call is refused until the next
 * _synthesize* or _run_frame_network call: the exported state carries no conditioning. */
LPCNET_EXPORT int lpcnet_b200_batch_synthesize_tail(LPCNetB200Batch *b, int samples, short *pcm, int preload);
/* run_frame_network_deferred / run_frame_network_flush (src/lpcnet.c:122-144): queue one feature frame per stream
 * (features [n_streams][feature_stride], at most 4 queued, older ones drop out) / run the frame network over the queue.
 * Each stream has its own queue: a reset or an import of a stream empties it, and the flush runs only the frames the stream
 * queued since.  The flush's conditioning is discarded; a later tail still reads that of the last frame-network run. */
LPCNET_EXPORT int lpcnet_b200_batch_frame_network_deferred(LPCNetB200Batch *b, const float *features, int feature_stride);
LPCNET_EXPORT int lpcnet_b200_batch_frame_network_flush(LPCNetB200Batch *b);

/* == state by value ==  The reference's PLC copies `LPCNetState` structs to roll back speculative synthesis
 * (src/lpcnet_plc.c:216-230).  One stream <-> opaque host blob of lpcnet_b200_batch_state_size() bytes (GRU states, signal
 * history, conv/LPC delay lines, decoder memory, RNG, frame counter).  The blob leaves out the conditioning a tail reads and
 * the deferred queue: exporting a stream with queued frames is refused, and an import empties the stream's queue and
 * refuses tails until the next frame-network run. */
LPCNET_EXPORT int lpcnet_b200_batch_state_size(const LPCNetB200Batch *b);
LPCNET_EXPORT int lpcnet_b200_batch_export_state(LPCNetB200Batch *b, int stream, void *buf);
LPCNET_EXPORT int lpcnet_b200_batch_import_state(LPCNetB200Batch *b, int stream, const void *buf);
/* ... and the whole batch, device to device, including what a tail reads and the deferred queues: */
LPCNET_EXPORT LPCNetB200Snapshot *lpcnet_b200_batch_snapshot_create(LPCNetB200Batch *b);
LPCNET_EXPORT void lpcnet_b200_batch_snapshot_destroy(LPCNetB200Snapshot *s);
LPCNET_EXPORT int lpcnet_b200_batch_snapshot_save(LPCNetB200Batch *b, LPCNetB200Snapshot *s);
LPCNET_EXPORT int lpcnet_b200_batch_snapshot_restore(LPCNetB200Batch *b, const LPCNetB200Snapshot *s);
/* ... and whole streams from rows of one batch to rows of another (or the same) batch, on the device: compacting a batch whose
 * sessions ended, rebalancing the shards of a multi-GPU job, cloning a stream.  For k < count: row dst_rows[k] of dst becomes,
 * bit for bit, what row src_rows[k] of src was before the call.  Copied: everything the exported blob carries (GRU states, signal
 * history, de-emphasis, last excitation, conv/LPC delay lines, decoder memory, RNG, frame counter), the stream's deferred frames
 * and its row of the conditioning a tail reads.  The source is unchanged; src == dst is allowed and every read sees the state
 * from before the call (a rotation of rows works); source rows may repeat (cloning); destination rows must be distinct.  Rows
 * not listed are untouched, their queues and tail conditioning included.
 * Tails: afterwards dst accepts _synthesize_tail only if it did before and src did too; otherwise it refuses tails until its next
 * frame-network run, as after an import.  The copied rows land in dst's current tail frame.  A copied stream with more queued
 * frames than dst's queue holds makes that queue longer at its old end, which the other streams never read.
 * Both batches must have the same GRU_A size, flavour (int8 / float) and switches (FEATURES_DELAY, END2END, LPC_GAMMA); weights are
 * not compared: a row copied between two models continues under dst's weights.  src and dst may be on different devices of this
 * process (peer DMA when the devices allow it, staged by the driver otherwise).  The call waits for all work queued on either
 * batch, on any CUDA stream, and returns when the copy is complete; later calls on either batch are ordered after it.
 * Returns -1 (message: lpcnet_b200_last_error) and changes nothing for a NULL argument, count < 0, a row out of range, a repeated
 * destination row or batches that do not match.  count == 0 does nothing and succeeds. */
LPCNET_EXPORT int lpcnet_b200_batch_copy_streams(LPCNetB200Batch *dst, const int *dst_rows, LPCNetB200Batch *src, const int *src_rows, int count);

/* == multi-GPU: PCM sink ==  Streams shard across GPUs with no data-path exchange (SURVEY.md 8e); the only transfer is the
 * gather of the PCM.  With a sink set, every synthesize/decode `_device` call also copies each finished chunk (<= 16 frames)
 * of its PCM to  sink[(first_row + s) * pitch_samples + t]  on a copy stream (DMA engines over NVLink, no SM time) while the next
 * chunk is being computed; the call's stream completes only after the last copy.  `sink` may live on another device of this
 * process (peer access) or in another process (lpcnet_b200_ipc_export on the owner, lpcnet_b200_ipc_open here).
 * sink == NULL removes it. */
LPCNET_EXPORT int lpcnet_b200_batch_set_pcm_sink(LPCNetB200Batch *b, short *sink, long long pitch_samples, long long first_row);
LPCNET_EXPORT int lpcnet_b200_ipc_export(void *d_ptr, unsigned char handle[64]);
LPCNET_EXPORT void *lpcnet_b200_ipc_open(const unsigned char handle[64]);
LPCNET_EXPORT int lpcnet_b200_ipc_close(void *p);
LPCNET_EXPORT int lpcnet_b200_set_device(int device);

/* == multi-GPU in ONE process ==  `n_streams` independent streams cut into contiguous index ranges over `n_devices` CUDA devices
 * (devices[k] = CUDA ordinal of shard k; NULL = 0..n_devices-1), weights replicated, one LPCNetB200Batch per device.  Every call
 * enqueues all shards (each on its device's own stream) and then waits: the devices run concurrently and nothing is exchanged
 * inside the sample loop.  Host-out calls let every device copy its shard to the caller's buffer over its own PCIe link;
 * `_gather` calls collect the PCM in the memory of devices[0] instead ([n_streams][T] int16, e.g. from lpcnet_b200_device_alloc_on):
 * each finished chunk travels by peer DMA over NVLink while the next chunk is computed (the PCM sink above).
 * Use pinned host buffers (lpcnet_b200_host_alloc) so that the copies of different devices overlap. */
typedef struct LPCNetB200Multi LPCNetB200Multi;
LPCNET_EXPORT LPCNetB200Multi *lpcnet_b200_multi_create(int n_streams, const unsigned char *blob, int blob_len, const LPCNetB200Config *cfg,
                                                        const int *devices, int n_devices);
LPCNET_EXPORT void lpcnet_b200_multi_destroy(LPCNetB200Multi *m);
LPCNET_EXPORT int lpcnet_b200_multi_streams(const LPCNetB200Multi *m);
LPCNET_EXPORT int lpcnet_b200_multi_devices(const LPCNetB200Multi *m);
/* 1 if every device can write devices[0]'s memory directly (NVLink peer access); 0: gathers are staged by the driver */
LPCNET_EXPORT int lpcnet_b200_multi_peer_access(const LPCNetB200Multi *m);
/* shard k: its CUDA device and stream range [first, first + count) */
LPCNET_EXPORT int lpcnet_b200_multi_shard(const LPCNetB200Multi *m, int k, int *device, int *first, int *count);
/* the shard's batch, for the per-stream lifecycle calls (reset_streams, export/import_state, snapshots) with LOCAL stream ids */
LPCNET_EXPORT LPCNetB200Batch *lpcnet_b200_multi_batch(LPCNetB200Multi *m, int k);
LPCNET_EXPORT int lpcnet_b200_multi_reset(LPCNetB200Multi *m);
LPCNET_EXPORT int lpcnet_b200_multi_set_codebooks(LPCNetB200Multi *m, const float *cb, size_t n_floats);
/* same arguments as lpcnet_b200_batch_synthesize / _decode with n = all streams */
LPCNET_EXPORT int lpcnet_b200_multi_synthesize(LPCNetB200Multi *m, const float *features, int nframes, int feature_stride,
                                               int samples_per_frame, short *pcm);
LPCNET_EXPORT int lpcnet_b200_multi_decode(LPCNetB200Multi *m, const unsigned char *packets, int npackets, short *pcm);
/* host in, PCM gathered on devices[0]: d_pcm [n_streams][nframes*samples_per_frame] (resp. [n_streams][npackets*640]) */
LPCNET_EXPORT int lpcnet_b200_multi_synthesize_gather(LPCNetB200Multi *m, const float *features, int nframes, int feature_stride,
                                                      int samples_per_frame, short *d_pcm);
LPCNET_EXPORT int lpcnet_b200_multi_decode_gather(LPCNetB200Multi *m, const unsigned char *packets, int npackets, short *d_pcm);
/* contiguous range of shard k when n items are cut into `parts` (sizes differ by at most one; earlier shards take the remainder) */
LPCNET_EXPORT int lpcnet_b200_shard_range(int n, int k, int parts, int *first, int *count);
LPCNET_EXPORT void *lpcnet_b200_device_alloc_on(int device, size_t bytes);
/* CUDA streams for the `cuda_stream` argument of the `_device` entry points (for callers without their own CUDA binding).
 * The engine orders its state across streams itself: consecutive calls may use different streams. */
LPCNET_EXPORT void *lpcnet_b200_stream_create(void);
LPCNET_EXPORT void lpcnet_b200_stream_destroy(void *stream);
LPCNET_EXPORT int lpcnet_b200_stream_sync(void *stream);

/* == lpcnet_decode() per stream, `npackets` times ==
 * packets: [n_streams][npackets][8] bytes ; pcm: [n_streams][npackets*640] int16
 * Decode and synthesis share one per-stream state, as lpcnet_decode() drives the LPCNetState inside LPCNetDecState: a decode
 * advances the frame counter by 4 per packet and leaves its last frame's conditioning for _synthesize_tail, and the decoder
 * memory carries from call to call (and through _export_state / _import_state and snapshots). */
LPCNET_EXPORT int lpcnet_b200_batch_decode(LPCNetB200Batch *b, const unsigned char *packets, int npackets, short *pcm);
LPCNET_EXPORT int lpcnet_b200_batch_decode_device(LPCNetB200Batch *b, const unsigned char *d_packets, int npackets,
                                                  short *d_pcm, void *cuda_stream);

/* == groups: several batches of one model shape in one per-sample launch ==
 * Several existing batches on ONE device with the same GRU_A size and one flavour (all int8 or all float), each at most once
 * (at most 16): their synthesize / decode calls run as one.  Each member runs its own frame network and its own silent-frame launches, then every
 * member's remaining frames take ONE per-sample kernel launch that spreads all members' streams over the SMs together (no
 * CTA holds streams of two members).  Group stream g = the streams of batches[0], then batches[1], ... in order (the sum of
 * their sizes); features, packets and PCM are laid out as for a batch of that many streams.
 * A group call leaves every member in exactly the state (PCM, recurrent state, RNG, frame counters, decoder memory, what a
 * later _synthesize_tail reads) the member's own call would leave it in on its rows of the inputs, from any member state.
 * The per-stream lifecycle calls (reset, tail, deferred / flush, export / import, snapshots, codebooks) stay on the members,
 * which keep their own switches (FEATURES_DELAY, END2END, LPC_GAMMA) and sparsity patterns.  Group calls are ordered with
 * the members' own calls like any other call, so `_device` group calls may be mixed with member calls on any stream.
 * A member with a PCM sink set is refused (multi-GPU groups below gather the PCM themselves).  The group does not own its members:
 * destroy the group before any member.
 * Float groups pick their kernel as a float batch does: the neuron-per-lane kernel while the plan's streams per CTA is at most
 * 4, the lane == stream kernel above that (or always, with LPCNET_B200_FLOAT_LANE_STREAM set at create).
 * group_create returns NULL (message: lpcnet_b200_last_error) for members on different devices, with different GRU_A
 * sizes, int8 and float members mixed, a member listed twice, or more than 16 members.  LPCNET_B200_STREAMS_PER_CTA is read
 * at create. */
typedef struct LPCNetB200Group LPCNetB200Group;
LPCNET_EXPORT LPCNetB200Group *lpcnet_b200_group_create(LPCNetB200Batch *const *batches, int count);
LPCNET_EXPORT void lpcnet_b200_group_destroy(LPCNetB200Group *g);
LPCNET_EXPORT int lpcnet_b200_group_streams(const LPCNetB200Group *g);
/* features [sum n][nframes][feature_stride] -> pcm [sum n][nframes*samples_per_frame] */
LPCNET_EXPORT int lpcnet_b200_group_synthesize(LPCNetB200Group *g, const float *features, int nframes, int feature_stride,
                                               int samples_per_frame, short *pcm);
LPCNET_EXPORT int lpcnet_b200_group_synthesize_device(LPCNetB200Group *g, const float *d_features, int nframes, int feature_stride,
                                                      int samples_per_frame, short *d_pcm, void *cuda_stream);
/* packets [sum n][npackets][8] -> pcm [sum n][npackets*640]; every member needs its codebooks */
LPCNET_EXPORT int lpcnet_b200_group_decode(LPCNetB200Group *g, const unsigned char *packets, int npackets, short *pcm);
LPCNET_EXPORT int lpcnet_b200_group_decode_device(LPCNetB200Group *g, const unsigned char *d_packets, int npackets, short *d_pcm,
                                                  void *cuda_stream);
/* Device time (ms) of the per-sample launches of the last group call: the fused launches and the members' silent-frame
 * launches (the latter until a member's next own call); *launches = engine kernels that call launched. */
LPCNET_EXPORT float lpcnet_b200_group_last_sample_kernel_ms(const LPCNetB200Group *g, int *launches);
/* Test hook (host only, no CUDA): the launch plan for members of n[count] streams on `sms` SMs.  *spc = the smallest streams
 * per CTA (1..32) for which sum ceil(n[k] / spc) <= sms, 32 if none; override_spc > 0 pins it (LPCNET_B200_STREAMS_PER_CTA).
 * Member k takes ceil(n[k] / spc) consecutive CTAs; *ctas = their total.  spc <= 16 selects the half-A-only schedule. */
LPCNET_EXPORT int lpcnet_b200_debug_group_plan(const int *n, int count, int sms, int override_spc, int *spc, int *ctas);
/* Test hook (host only, no CUDA): the launch plan of a float group.  *spc as above; then, as for a float batch, spc <= 4 with
 * lane_stream 0 selects the neuron-per-lane kernel, whose CTAs lay out *slots = 1, 2 or 4 streams (spc 3 -> 4), and anything
 * else the lane == stream kernel with *slots = spc.  Member k takes ceil(n[k] / slots) consecutive CTAs; *ctas = their total.
 * lane_stream != 0 stands for LPCNET_B200_FLOAT_LANE_STREAM.  Returns 1 for the neuron-per-lane kernel, 0 for the lane == stream
 * kernel, -1 for bad arguments. */
LPCNET_EXPORT int lpcnet_b200_debug_group_plan_float(const int *n, int count, int sms, int override_spc, int lane_stream,
                                                     int *spc, int *slots, int *ctas);

/* == mixed groups: batches of different GRU_A sizes and flavours in one call ==
 * 1..16 existing batches on ONE device, each at most once, of any GRU_A size (128, 256, 384) and either flavour.  Members are
 * partitioned into classes by (GRU_A size, flavour), in order of first appearance, and each class is one ordinary group
 * (lpcnet_b200_group_create's kernel, CTA layout and shared memory) over its members in member order.  All classes share one
 * streams-per-CTA value: the one a group over ALL members would plan (lpcnet_b200_debug_group_plan: the smallest spc at which
 * sum ceil(n_k / spc) <= SM count, 32 if none; LPCNET_B200_STREAMS_PER_CTA pins it), so that the classes' CTAs together fit on the
 * SMs (a float class's CTAs lay out slots >= spc streams, see lpcnet_b200_debug_group_plan_float).  A one-shape member list plans
 * exactly as its group.  LPCNET_B200_STREAMS_PER_CTA and LPCNET_B200_FLOAT_LANE_STREAM are read at create.
 * A call checks every class as that class's group call would, and refuses before anything is enqueued on any stream.  It then
 * runs class 0's group call on the call's stream and every other class's on a stream the mixed group owns, forked from the call's
 * stream and joined back into it, so the classes' per-sample launches can run at the same time on disjoint SMs.  Whether they do
 * is up to the hardware; results never depend on it.
 * Mixed-group stream g = the streams of batches[0], then batches[1], ... in order; features, packets and PCM are laid out as for a
 * batch of that many streams.  The contract is the group's: a call leaves every member in exactly the state its own call on its
 * rows of the inputs would leave it in (PCM, recurrent state, RNG, frame counters, decoder memory, what a later tail reads), from
 * any member state.  Calls are ordered with every other call on the members, so `_device` calls may be mixed with member calls,
 * ordinary groups over the same batches and the members' lifecycle calls on any stream.  A member with a PCM sink is refused,
 * as is a decode with a member that has no codebooks.
 * create returns NULL (message: lpcnet_b200_last_error) for a NULL argument, count outside 1..16, a member listed twice or
 * members on different devices.  The mixed group does not own its members: destroy it before any of them. */
typedef struct LPCNetB200MixedGroup LPCNetB200MixedGroup;
LPCNET_EXPORT LPCNetB200MixedGroup *lpcnet_b200_mixed_group_create(LPCNetB200Batch *const *batches, int count);
LPCNET_EXPORT void lpcnet_b200_mixed_group_destroy(LPCNetB200MixedGroup *mg);
LPCNET_EXPORT int lpcnet_b200_mixed_group_streams(const LPCNetB200MixedGroup *mg);
LPCNET_EXPORT int lpcnet_b200_mixed_group_classes(const LPCNetB200MixedGroup *mg);
/* class c's group (lpcnet_b200_group_last_sample_kernel_ms of its part of the last call, introspection); owned by the mixed group */
LPCNET_EXPORT LPCNetB200Group *lpcnet_b200_mixed_group_group(LPCNetB200MixedGroup *mg, int c);
/* features [sum n][nframes][feature_stride] -> pcm [sum n][nframes*samples_per_frame] */
LPCNET_EXPORT int lpcnet_b200_mixed_group_synthesize(LPCNetB200MixedGroup *mg, const float *features, int nframes, int feature_stride,
                                                     int samples_per_frame, short *pcm);
LPCNET_EXPORT int lpcnet_b200_mixed_group_synthesize_device(LPCNetB200MixedGroup *mg, const float *d_features, int nframes,
                                                            int feature_stride, int samples_per_frame, short *d_pcm, void *cuda_stream);
/* packets [sum n][npackets][8] -> pcm [sum n][npackets*640]; every member needs its codebooks */
LPCNET_EXPORT int lpcnet_b200_mixed_group_decode(LPCNetB200MixedGroup *mg, const unsigned char *packets, int npackets, short *pcm);
LPCNET_EXPORT int lpcnet_b200_mixed_group_decode_device(LPCNetB200MixedGroup *mg, const unsigned char *d_packets, int npackets,
                                                        short *d_pcm, void *cuda_stream);
/* device time (ms) of the last call, from the fork on the call's stream to the join of every class (<0 on error, 0 before any call) */
LPCNET_EXPORT float lpcnet_b200_mixed_group_last_call_ms(const LPCNetB200MixedGroup *mg);
/* Test hook (host only, no CUDA): the plan of a mixed group whose member k has n[k] streams, na[k] GRU_A units and flavour is_float[k]
 * (0 / 1) on `sms` SMs.  *spc as lpcnet_b200_debug_group_plan over all members; class_of[k] = member k's class; per class c:
 * class_ctas[c] = its CTAs (int8: sum ceil(n_k / spc); float: sum ceil(n_k / slots), slots as lpcnet_b200_debug_group_plan_float) and
 * class_neuron[c] = 1 for a float class on the neuron-per-lane kernel.  lane_stream != 0 stands for LPCNET_B200_FLOAT_LANE_STREAM.
 * Returns the number of classes, -1 for bad arguments. */
LPCNET_EXPORT int lpcnet_b200_debug_mixed_plan(const int *n, const int *na, const int *is_float, int count, int sms, int override_spc,
                                               int lane_stream, int *spc, int *class_of, int *class_ctas, int *class_neuron);

/* == multi-GPU groups: several models over every GPU of the process in one call ==
 * The members are existing multi-GPU objects (lpcnet_b200_multi_create), one per model, all over the same device list in the same
 * order, with one GRU_A size and one flavour (all int8 or all float), each at most once (at most 16).  Each keeps its own stream
 * count and sharding; shard k of every member sits on devices[k].  For each device the multi-group holds one group
 * (lpcnet_b200_group_create) over that device's shard batches, in member order, so every device runs each member's frame
 * network and silent-frame launches, then one per-sample launch per chunk for all of them.  Every call enqueues all devices, each
 * on a stream of its own, then waits for all of them.
 * Job row r = member 0's streams in its own order, then member 1's, ... (the sum of their sizes, lpcnet_b200_multi_group_streams);
 * features, packets and PCM are laid out as for lpcnet_b200_multi_* with that many streams.  `_gather` calls collect the PCM in the
 * memory of devices[0] ([sum n][T] int16): every finished chunk (<= 16 frames) of every member's shard travels to its rows there
 * on a copy stream (peer DMA when lpcnet_b200_multi_peer_access allows it, staged by the driver otherwise) while the next chunk is
 * computed; the call returns once the gathered PCM is complete.  As for lpcnet_b200_multi_*, pinned host buffers
 * (lpcnet_b200_host_alloc) let the copies of different devices overlap.
 * A call leaves every member exactly as the member's own lpcnet_b200_multi_synthesize / _decode on its rows of the inputs would:
 * PCM, recurrent state, RNG, frame counters, decoder memory, what a later tail reads.  Multi-group calls are ordered with every
 * other call on the shard batches, so they may be mixed with member multi calls, shard lifecycle calls (reset_streams,
 * export / import, copy_streams) and single-device group calls over the shards.  A PCM sink a member's own `_gather` call left on a
 * shard batch is neither used nor cleared.  Bad arguments (feature_stride < 20, samples_per_frame outside 1..65536, a decode
 * with a member that has no codebooks) are refused before anything is enqueued on any device.
 * create returns NULL (message: lpcnet_b200_last_error) and changes nothing for a NULL argument, count outside 1..16, a member
 * listed twice, members over different device lists, different GRU_A sizes, or int8 and float members mixed.  The multi-group
 * does not own its members: destroy it before any of them. */
typedef struct LPCNetB200MultiGroup LPCNetB200MultiGroup;
LPCNET_EXPORT LPCNetB200MultiGroup *lpcnet_b200_multi_group_create(LPCNetB200Multi *const *members, int count);
LPCNET_EXPORT void lpcnet_b200_multi_group_destroy(LPCNetB200MultiGroup *mg);
LPCNET_EXPORT int lpcnet_b200_multi_group_streams(const LPCNetB200MultiGroup *mg);
/* the group of devices[k] (lpcnet_b200_group_last_sample_kernel_ms of that device's last call, introspection) */
LPCNET_EXPORT LPCNetB200Group *lpcnet_b200_multi_group_group(LPCNetB200MultiGroup *mg, int k);
/* features [sum n][nframes][feature_stride] -> pcm [sum n][nframes*samples_per_frame] on the host / gathered on devices[0] */
LPCNET_EXPORT int lpcnet_b200_multi_group_synthesize(LPCNetB200MultiGroup *mg, const float *features, int nframes, int feature_stride,
                                                     int samples_per_frame, short *pcm);
LPCNET_EXPORT int lpcnet_b200_multi_group_synthesize_gather(LPCNetB200MultiGroup *mg, const float *features, int nframes,
                                                            int feature_stride, int samples_per_frame, short *d_pcm);
/* packets [sum n][npackets][8] -> pcm [sum n][npackets*640]; every member needs its codebooks */
LPCNET_EXPORT int lpcnet_b200_multi_group_decode(LPCNetB200MultiGroup *mg, const unsigned char *packets, int npackets, short *pcm);
LPCNET_EXPORT int lpcnet_b200_multi_group_decode_gather(LPCNetB200MultiGroup *mg, const unsigned char *packets, int npackets, short *d_pcm);

/* == the analysis side, batched (SURVEY 8f N2): feature extraction and the 1.6 kb/s encoder ==
 * n independent LPCNetEncState streams (reference src/lpcnet_private.h:55-75) on one device, all starting from
 * lpcnet_encoder_create() (zeroed state, src/lpcnet_enc.c:471-482).  Results equal the reference's per-stream calls.
 * As with a synthesis batch, consecutive `_device` calls may use different CUDA streams and may be mixed with host calls. */
typedef struct LPCNetB200EncBatch LPCNetB200EncBatch;
LPCNET_EXPORT LPCNetB200EncBatch *lpcnet_b200_enc_create(int n_streams, int device);
LPCNET_EXPORT void lpcnet_b200_enc_destroy(LPCNetB200EncBatch *e);
LPCNET_EXPORT int lpcnet_b200_enc_reset(LPCNetB200EncBatch *e);                      /* lpcnet_encoder_init() for every stream */
LPCNET_EXPORT int lpcnet_b200_enc_streams(const LPCNetB200EncBatch *e);
/* == per-stream state ==  A row is its whole LPCNetEncState: analysis memory, pre-emphasis memory, pcount (the sub-frame slot),
 * the pitch history, xc and frame weights, the excitation buffer, the Viterbi paths, best_i, vq_mem and the four-frame feature
 * buffer.  What a row produces after a reset, an import or a copy equals, bit for bit, what the reference produces from that
 * state, also for a row caught mid-superframe (pcount != 0 after single-frame calls).
 * Every call below waits for all work queued on the batches it touches, on any CUDA stream, and returns when its work is
 * complete; later calls on those batches, `_device` calls on caller streams included, are ordered after it.  Each returns -1
 * (message: lpcnet_b200_last_error) and changes nothing for a NULL argument, count < 0 or a row out of range; count == 0 does
 * nothing and succeeds. */
/* lpcnet_encoder_init() for the listed streams only; the other streams carry on.  Ids may repeat. */
LPCNET_EXPORT int lpcnet_b200_enc_reset_streams(LPCNetB200EncBatch *e, const int *streams, int count);
/* One stream <-> opaque host blob of lpcnet_b200_enc_state_size() bytes: everything a later call reads.  An import validates
 * the blob on the host first and refuses one whose pcount is outside 0..3 or whose best_i is outside 0..255. */
LPCNET_EXPORT int lpcnet_b200_enc_state_size(const LPCNetB200EncBatch *e);
LPCNET_EXPORT int lpcnet_b200_enc_export_state(LPCNetB200EncBatch *e, int stream, void *buf);
LPCNET_EXPORT int lpcnet_b200_enc_import_state(LPCNetB200EncBatch *e, int stream, const void *buf);
/* Row dst_rows[k] of dst becomes, bit for bit, what row src_rows[k] of src was before the call (compacting a batch whose
 * sessions ended, moving a session to another batch or GPU, forking one).  The source is unchanged; src == dst is allowed and
 * every read sees the state from before the call (a rotation of rows works); source rows may repeat (cloning); destination
 * rows must be distinct (a repeated one is refused like a row out of range).  Rows not listed are untouched.  Codebooks are
 * not compared: a copied row goes on under dst's codebooks, and dst without codebooks still refuses _encode.  src and dst may
 * be on different devices of this process (peer DMA when the devices allow it, staged by the driver otherwise). */
LPCNET_EXPORT int lpcnet_b200_enc_copy_streams(LPCNetB200EncBatch *dst, const int *dst_rows,
                                               LPCNetB200EncBatch *src, const int *src_rows, int count);
/* the VQ codebooks lpcnet_encode searches (same four arrays, same order as lpcnet_b200_batch_set_codebooks) */
LPCNET_EXPORT int lpcnet_b200_enc_set_codebooks(LPCNetB200EncBatch *e, const float *cb, size_t n_floats);
/* == lpcnet_compute_single_frame_features() per stream and frame (src/lpcnet_enc.c:919; `lpcnet_demo -features`) ==
 * pcm [n_streams][nframes*160] int16 (or float: lpcnet_compute_single_frame_features_float) -> features [n_streams][nframes][36]
 * (18 cepstral coefficients, pitch, pitch correlation, 16 LPC: the `.f32` feature-file row the synthesis side reads) */
LPCNET_EXPORT int lpcnet_b200_enc_compute_features(LPCNetB200EncBatch *e, const short *pcm, int nframes, float *features);
LPCNET_EXPORT int lpcnet_b200_enc_compute_features_float(LPCNetB200EncBatch *e, const float *pcm, int nframes, float *features);
LPCNET_EXPORT int lpcnet_b200_enc_compute_features_device(LPCNetB200EncBatch *e, const short *d_pcm, int nframes, float *d_features, void *cuda_stream);
/* == lpcnet_encode() per stream and 640-sample packet (src/lpcnet_enc.c:882) ==  pcm [n][npackets*640] -> packets [n][npackets][8] */
LPCNET_EXPORT int lpcnet_b200_enc_encode(LPCNetB200EncBatch *e, const short *pcm, int npackets, unsigned char *packets);
LPCNET_EXPORT int lpcnet_b200_enc_encode_device(LPCNetB200EncBatch *e, const short *d_pcm, int npackets, unsigned char *d_packets, void *cuda_stream);
/* == lpcnet_compute_features() (src/lpcnet_enc.c:896): unquantised 4-frame analysis ==  pcm [n][npackets*640] -> features [n][npackets*4][36] */
LPCNET_EXPORT int lpcnet_b200_enc_compute_features4(LPCNetB200EncBatch *e, const short *pcm, int npackets, float *features);
/* Test hook (host only): the analysis window and DCT table as the engine builds them (src/dump_lpcnet_tables.c:83-96): hw[160], dct[324] */
LPCNET_EXPORT void lpcnet_b200_enc_tables(float *half_window, float *dct);

/* ---- introspection used by the tests and the benchmark ---- */
/* Device time (ms, CUDA events on the engine's stream) the per-sample kernel took in the last synthesize/decode
 * call, summed over its launches; *launches receives how many engine kernels that call launched in total. */
LPCNET_EXPORT float lpcnet_b200_batch_last_sample_kernel_ms(const LPCNetB200Batch *b, int *launches);
/* CUDA-event stopwatch on the engine's stream, L2 eviction (256 MiB overwrite) and stream sync: what a benchmark
 * needs to time the engine on the device without any other CUDA binding. */
LPCNET_EXPORT int lpcnet_b200_batch_timer_start(LPCNetB200Batch *b);
LPCNET_EXPORT float lpcnet_b200_batch_timer_stop(LPCNetB200Batch *b);     /* ms since timer_start, <0 on error */
LPCNET_EXPORT int lpcnet_b200_batch_flush_l2(LPCNetB200Batch *b);
LPCNET_EXPORT int lpcnet_b200_batch_sync(LPCNetB200Batch *b);
/* Raw device / pinned-host memory for callers without their own CUDA binding. */
LPCNET_EXPORT void *lpcnet_b200_device_alloc(size_t bytes);
LPCNET_EXPORT void lpcnet_b200_device_free(void *p);
LPCNET_EXPORT int lpcnet_b200_memcpy_h2d(void *dst, const void *src, size_t bytes);
LPCNET_EXPORT int lpcnet_b200_memcpy_d2h(void *dst, const void *src, size_t bytes);
LPCNET_EXPORT void *lpcnet_b200_host_alloc(size_t bytes);                 /* pinned */
LPCNET_EXPORT void lpcnet_b200_host_free(void *p);

/* Measured peak of the unit that bounds the per-sample kernel, the L1/shared-memory data pipe: every SM streams
 * conflict-free LDS out of shared memory (lpcnet_b200/csrc/microbench.cu).  out[7] = {LDS.128 GB/s whole chip,
 * LDS.128 bytes/clk/SM, LDS.64 GB/s, LDS.64 B/clk/SM, LDS.32 GB/s, LDS.32 B/clk/SM, SM count}. */
LPCNET_EXPORT int lpcnet_b200_measure_smem_peak(int device, double *out);

/* Algorithmic bytes one synthesized sample of one stream must read (SURVEY.md 8d): total and the
 * sparse-GEMV-only subset (GRU_A weights + indices). */
LPCNET_EXPORT int lpcnet_b200_batch_algorithmic_bytes(const LPCNetB200Batch *b, long *total, long *sparse_gemv);
/* 1 if the loaded blob is the float (DISABLE_DOT_PROD) flavour, 0 for int8. */
LPCNET_EXPORT int lpcnet_b200_batch_is_float(const LPCNetB200Batch *b);
/* Copy the per-stream recurrent state of stream `s` to host (tests): gru_a[384], gru_b[16], last_sig[16],
 * misc[2]={last_exc, frame_count}, rng[4]. Any pointer may be NULL. */
LPCNET_EXPORT int lpcnet_b200_batch_get_state(LPCNetB200Batch *b, int s, float *gru_a, float *gru_b, float *last_sig,
                                              int *misc, uint32_t *rng);
/* Frame-network tap (tests): run ONLY the 100 Hz kernels (reference run_frame_network, src/lpcnet.c:82-120) on
 * host features [n][nframes<=16][feature_stride] and return gru_a_condition [n][nframes][1152], gru_b_condition
 * [n][nframes][48] and the gamma-weighted LPC [n][nframes][16] each frame's sample loop would use. */
LPCNET_EXPORT int lpcnet_b200_debug_frame_network(LPCNetB200Batch *b, const float *features, int nframes,
                                                  int feature_stride, float *ga, float *gb, float *lpc);
/* Test hook (host only, no CUDA): build the per-sample kernel's shared-memory image for a blob.  Returns the
 * image size or <0; layout[24] receives the offsets documented in lpcnet_b200/csrc/batch_api.cu. */
LPCNET_EXPORT int lpcnet_b200_debug_image(const unsigned char *blob, int len, unsigned char *out, size_t cap,
                                          uint32_t *layout);

/* Same for the second image of float models (the neuron-per-lane kernel used for small batches); layout[17]. */
LPCNET_EXPORT int lpcnet_b200_debug_image_n(const unsigned char *blob, int len, unsigned char *out, size_t cap,
                                            uint32_t *layout);
/* Test hook: evaluate the engine's emulation of the reference's _mm256_rcp_ps (the per-sample kernels' table) on n host
 * floats. */
LPCNET_EXPORT int lpcnet_b200_debug_rcp(LPCNetB200Batch *b, const float *x, float *out, int n);
/* Test hook: the conditioning network's full-range _mm256_rcp_ps emulation (zeros, denormals, infinities, NaN, |x| >= 2^126)
 * and its tanh8_approx with the reference's NaN order on n host floats. */
LPCNET_EXPORT int lpcnet_b200_debug_tanh_x86(LPCNetB200Batch *b, const float *x, float *out_rcp, float *out_tanh, int n);

/* Default model / codebooks for the lpcnet.h single-stream API (the reference compiles its model in; this
 * library loads it at run time).  Also settable through env LPCNET_B200_MODEL / LPCNET_B200_CODEBOOKS (file
 * paths) and LPCNET_B200_LPC_GAMMA. */
LPCNET_EXPORT int lpcnet_b200_set_default_model(const unsigned char *blob, int len, float lpc_gamma);
LPCNET_EXPORT int lpcnet_b200_set_default_codebooks(const float *cb, size_t n_floats);
/* Release the device resources behind a state that was set up with lpcnet_init() / lpcnet_decoder_init() on
 * caller-owned memory (reference include/lpcnet.h:160-169: get_size + init, no matching deinit).  Without this call they
 * are released at process exit, or when the same memory is initialised again.  `st` is the LPCNetState* (a
 * LPCNetDecState* may be passed as well: it starts with its LPCNetState, src/lpcnet_private.h:50-53). */
struct LPCNetState;
LPCNET_EXPORT void lpcnet_b200_deinit(struct LPCNetState *st);

#ifdef __cplusplus
}
#endif
#endif
