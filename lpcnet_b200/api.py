import ctypes
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("LPCNET_B200_SO") or os.path.join(_HERE, "liblpcnet_b200.so")   # env override: tuning variants only
c_p = ctypes.c_void_p


class LPCNetB200Error(RuntimeError):
    pass


_lib = None


def lib():
    """Load liblpcnet_b200.so (built in-tree by lpcnet_b200.build).  Fails loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise LPCNetB200Error("liblpcnet_b200.so is not built (run `python -m lpcnet_b200.build`); there is no fallback path")
    L = ctypes.CDLL(_SO)
    L.lpcnet_b200_last_error.restype = ctypes.c_char_p
    L.lpcnet_b200_batch_create.restype = c_p
    L.lpcnet_b200_batch_create.argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_float, ctypes.c_int]
    L.lpcnet_b200_batch_create_ex.restype = c_p
    L.lpcnet_b200_batch_create_ex.argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int]
    L.lpcnet_b200_batch_model_info.argtypes = [c_p, c_p, c_p]
    L.lpcnet_b200_batch_reset_streams.argtypes = [c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_batch_reset_signal.argtypes = [c_p]
    L.lpcnet_b200_batch_synthesize_ex.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, ctypes.c_int]
    L.lpcnet_b200_batch_synthesize_device_ex.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_batch_run_frame_network.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int]
    L.lpcnet_b200_batch_synthesize_tail.argtypes = [c_p, ctypes.c_int, c_p, ctypes.c_int]
    L.lpcnet_b200_batch_frame_network_deferred.argtypes = [c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_batch_frame_network_flush.argtypes = [c_p]
    L.lpcnet_b200_batch_state_size.argtypes = [c_p]
    L.lpcnet_b200_batch_export_state.argtypes = [c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_batch_import_state.argtypes = [c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_batch_snapshot_create.restype = c_p
    L.lpcnet_b200_batch_snapshot_create.argtypes = [c_p]
    L.lpcnet_b200_batch_snapshot_destroy.argtypes = [c_p]
    L.lpcnet_b200_batch_snapshot_save.argtypes = [c_p, c_p]
    L.lpcnet_b200_batch_snapshot_restore.argtypes = [c_p, c_p]
    L.lpcnet_b200_batch_copy_streams.argtypes = [c_p, c_p, c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_batch_set_pcm_sink.argtypes = [c_p, c_p, ctypes.c_longlong, ctypes.c_longlong]
    L.lpcnet_b200_ipc_export.argtypes = [c_p, c_p]
    L.lpcnet_b200_ipc_open.restype = c_p
    L.lpcnet_b200_ipc_open.argtypes = [c_p]
    L.lpcnet_b200_ipc_close.argtypes = [c_p]
    L.lpcnet_b200_set_device.argtypes = [ctypes.c_int]
    L.lpcnet_b200_stream_create.restype = c_p
    L.lpcnet_b200_stream_destroy.argtypes = [c_p]
    L.lpcnet_b200_stream_sync.argtypes = [c_p]
    L.lpcnet_b200_batch_destroy.argtypes = [c_p]
    L.lpcnet_b200_batch_reset.argtypes = [c_p]
    L.lpcnet_b200_batch_streams.argtypes = [c_p]
    L.lpcnet_b200_batch_set_codebooks.argtypes = [c_p, c_p, ctypes.c_size_t]
    L.lpcnet_b200_batch_synthesize.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_batch_synthesize_device.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_batch_decode.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_batch_decode_device.argtypes = [c_p, c_p, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_batch_last_sample_kernel_ms.restype = ctypes.c_float
    L.lpcnet_b200_batch_last_sample_kernel_ms.argtypes = [c_p, c_p]
    L.lpcnet_b200_batch_algorithmic_bytes.argtypes = [c_p, c_p, c_p]
    # groups of batches (one per-sample launch for several models of one shape)
    L.lpcnet_b200_group_create.restype = c_p
    L.lpcnet_b200_group_create.argtypes = [c_p, ctypes.c_int]
    L.lpcnet_b200_group_destroy.argtypes = [c_p]
    L.lpcnet_b200_group_streams.argtypes = [c_p]
    L.lpcnet_b200_group_synthesize.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_group_synthesize_device.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_group_decode.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_group_decode_device.argtypes = [c_p, c_p, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_group_last_sample_kernel_ms.restype = ctypes.c_float
    L.lpcnet_b200_group_last_sample_kernel_ms.argtypes = [c_p, c_p]
    L.lpcnet_b200_debug_group_plan.argtypes = [c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_debug_group_plan_float.argtypes = [c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p, c_p]
    # mixed groups (several group shapes, one launch per shape on streams of their own)
    L.lpcnet_b200_mixed_group_create.restype = c_p
    L.lpcnet_b200_mixed_group_create.argtypes = [c_p, ctypes.c_int]
    L.lpcnet_b200_mixed_group_destroy.argtypes = [c_p]
    L.lpcnet_b200_mixed_group_streams.argtypes = [c_p]
    L.lpcnet_b200_mixed_group_classes.argtypes = [c_p]
    L.lpcnet_b200_mixed_group_group.restype = c_p
    L.lpcnet_b200_mixed_group_group.argtypes = [c_p, ctypes.c_int]
    L.lpcnet_b200_mixed_group_synthesize.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_mixed_group_synthesize_device.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_mixed_group_decode.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_mixed_group_decode_device.argtypes = [c_p, c_p, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_mixed_group_last_call_ms.restype = ctypes.c_float
    L.lpcnet_b200_mixed_group_last_call_ms.argtypes = [c_p]
    L.lpcnet_b200_debug_mixed_plan.argtypes = [c_p, c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p, c_p, c_p]
    L.lpcnet_b200_batch_is_float.argtypes = [c_p]
    L.lpcnet_b200_batch_get_state.argtypes = [c_p, ctypes.c_int, c_p, c_p, c_p, c_p, c_p]
    L.lpcnet_b200_debug_frame_network.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, c_p, c_p, c_p]
    L.lpcnet_b200_debug_rcp.argtypes = [c_p, c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_debug_tanh_x86.argtypes = [c_p, c_p, c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_set_default_model.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_float]
    L.lpcnet_b200_set_default_codebooks.argtypes = [c_p, ctypes.c_size_t]
    L.lpcnet_b200_batch_timer_start.argtypes = [c_p]
    L.lpcnet_b200_batch_timer_stop.restype = ctypes.c_float
    L.lpcnet_b200_batch_timer_stop.argtypes = [c_p]
    L.lpcnet_b200_batch_flush_l2.argtypes = [c_p]
    L.lpcnet_b200_batch_sync.argtypes = [c_p]
    L.lpcnet_b200_device_alloc.restype = c_p
    L.lpcnet_b200_device_alloc.argtypes = [ctypes.c_size_t]
    L.lpcnet_b200_device_free.argtypes = [c_p]
    L.lpcnet_b200_memcpy_h2d.argtypes = [c_p, c_p, ctypes.c_size_t]
    L.lpcnet_b200_memcpy_d2h.argtypes = [c_p, c_p, ctypes.c_size_t]
    L.lpcnet_b200_host_alloc.restype = c_p
    L.lpcnet_b200_host_alloc.argtypes = [ctypes.c_size_t]
    L.lpcnet_b200_host_free.argtypes = [c_p]
    L.lpcnet_b200_measure_smem_peak.argtypes = [ctypes.c_int, c_p]
    # model blob I/O (csrc/blob_io.cu)
    L.lpcnet_b200_write_blob.restype = ctypes.c_longlong
    L.lpcnet_b200_write_blob.argtypes = [c_p, ctypes.c_int, c_p, c_p, ctypes.c_size_t]
    L.lpcnet_b200_write_blob_file.argtypes = [ctypes.c_char_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_parse_blob.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int]
    L.lpcnet_b200_blob_config.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p]
    L.lpcnet_b200_read_file.restype = ctypes.c_longlong
    L.lpcnet_b200_read_file.argtypes = [ctypes.c_char_p, c_p, ctypes.c_size_t]
    # multi-GPU in one process (csrc/multi_api.cu)
    L.lpcnet_b200_multi_create.restype = c_p
    L.lpcnet_b200_multi_create.argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_int, c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_multi_destroy.argtypes = [c_p]
    L.lpcnet_b200_multi_streams.argtypes = [c_p]
    L.lpcnet_b200_multi_devices.argtypes = [c_p]
    L.lpcnet_b200_multi_peer_access.argtypes = [c_p]
    L.lpcnet_b200_multi_shard.argtypes = [c_p, ctypes.c_int, c_p, c_p, c_p]
    L.lpcnet_b200_multi_batch.restype = c_p
    L.lpcnet_b200_multi_batch.argtypes = [c_p, ctypes.c_int]
    L.lpcnet_b200_multi_reset.argtypes = [c_p]
    L.lpcnet_b200_multi_set_codebooks.argtypes = [c_p, c_p, ctypes.c_size_t]
    L.lpcnet_b200_multi_synthesize.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_multi_decode.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_multi_synthesize_gather.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_multi_decode_gather.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_shard_range.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_device_alloc_on.restype = c_p
    L.lpcnet_b200_device_alloc_on.argtypes = [ctypes.c_int, ctypes.c_size_t]
    L.lpcnet_b200_multi_group_create.restype = c_p
    L.lpcnet_b200_multi_group_create.argtypes = [c_p, ctypes.c_int]
    L.lpcnet_b200_multi_group_destroy.argtypes = [c_p]
    L.lpcnet_b200_multi_group_streams.argtypes = [c_p]
    L.lpcnet_b200_multi_group_group.restype = c_p
    L.lpcnet_b200_multi_group_group.argtypes = [c_p, ctypes.c_int]
    L.lpcnet_b200_multi_group_synthesize.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_multi_group_synthesize_gather.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.lpcnet_b200_multi_group_decode.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_multi_group_decode_gather.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    # analysis side (csrc/enc_kernels.cu)
    L.lpcnet_b200_enc_create.restype = c_p
    L.lpcnet_b200_enc_create.argtypes = [ctypes.c_int, ctypes.c_int]
    L.lpcnet_b200_enc_destroy.argtypes = [c_p]
    L.lpcnet_b200_enc_reset.argtypes = [c_p]
    L.lpcnet_b200_enc_streams.argtypes = [c_p]
    L.lpcnet_b200_enc_reset_streams.argtypes = [c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_enc_state_size.argtypes = [c_p]
    L.lpcnet_b200_enc_export_state.argtypes = [c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_enc_import_state.argtypes = [c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_enc_copy_streams.argtypes = [c_p, c_p, c_p, c_p, ctypes.c_int]
    L.lpcnet_b200_enc_set_codebooks.argtypes = [c_p, c_p, ctypes.c_size_t]
    L.lpcnet_b200_enc_compute_features.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_enc_compute_features_float.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_enc_compute_features_device.argtypes = [c_p, c_p, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_enc_encode.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_enc_encode_device.argtypes = [c_p, c_p, ctypes.c_int, c_p, c_p]
    L.lpcnet_b200_enc_compute_features4.argtypes = [c_p, c_p, ctypes.c_int, c_p]
    L.lpcnet_b200_enc_tables.restype = None
    L.lpcnet_b200_enc_tables.argtypes = [c_p, c_p]
    # reference API (include/lpcnet.h)
    L.lpcnet_create.restype = c_p
    L.lpcnet_destroy.argtypes = [c_p]
    L.lpcnet_init.argtypes = [c_p]
    L.lpcnet_reset.argtypes = [c_p]
    L.lpcnet_load_model.argtypes = [c_p, ctypes.c_char_p, ctypes.c_int]
    L.lpcnet_synthesize.restype = None
    L.lpcnet_synthesize.argtypes = [c_p, c_p, c_p, ctypes.c_int]
    L.lpcnet_decoder_create.restype = c_p
    L.lpcnet_decoder_destroy.argtypes = [c_p]
    L.lpcnet_decoder_init.argtypes = [c_p]
    L.lpcnet_decode.argtypes = [c_p, c_p, c_p]
    _lib = L
    return L


def _err():
    return (lib().lpcnet_b200_last_error() or b"").decode()


def device_count():
    return lib().lpcnet_b200_device_count()


def measure_smem_peak(device=0):
    """Measured shared-memory streaming peak (conflict-free LDS on every SM): dict of GB/s and bytes/clk/SM per width."""
    out = (ctypes.c_double * 7)()
    if lib().lpcnet_b200_measure_smem_peak(int(device), out) != 0:
        raise LPCNetB200Error("measure_smem_peak: " + _err())
    return {"lds128_gbs": out[0], "lds128_bytes_per_clk_sm": out[1], "lds64_gbs": out[2], "lds64_bytes_per_clk_sm": out[3],
            "lds32_gbs": out[4], "lds32_bytes_per_clk_sm": out[5], "sms": int(out[6])}


class Config(ctypes.Structure):
    """LPCNetB200Config (include/lpcnet_b200.h): LPC_GAMMA / FEATURES_DELAY / END2END of the model's generated nnet_data.h."""
    _fields_ = [("lpc_gamma", ctypes.c_float), ("features_delay", ctypes.c_int), ("end2end", ctypes.c_int)]


class Array(ctypes.Structure):
    """LPCNetB200Array (include/lpcnet_b200.h) = the reference's WeightArray (src/nnet.h:43-48)."""
    _fields_ = [("name", ctypes.c_char_p), ("type", ctypes.c_int), ("size", ctypes.c_int), ("data", ctypes.c_void_p)]


def parse_blob(blob):
    """[(name, type, bytes)] of a DNNw blob (lpcnet_b200_parse_blob)."""
    L = lib()
    n = L.lpcnet_b200_parse_blob(blob, len(blob), None, 0)
    if n < 0:
        raise LPCNetB200Error("parse_blob: " + _err())
    recs = (Array * n)()
    L.lpcnet_b200_parse_blob(blob, len(blob), recs, n)
    return [(r.name.decode(), int(r.type), ctypes.string_at(r.data, r.size)) for r in recs]


def write_blob(arrays, config=None):
    """arrays: [(name, type, bytes-like)] -> DNNw blob bytes (lpcnet_b200_write_blob); config = (gamma, delay, end2end) or None."""
    L = lib()
    n = len(arrays)
    recs = (Array * n)()
    keep = []
    for i, (name, typ, data) in enumerate(arrays):
        raw = bytes(data)
        buf = ctypes.create_string_buffer(raw, len(raw))
        nm = name.encode()
        keep += [buf, nm]
        recs[i].name = nm; recs[i].type = int(typ); recs[i].size = len(raw); recs[i].data = ctypes.addressof(buf)
    c = Config(float(config[0]), int(config[1]), int(config[2])) if config is not None else None
    cp = ctypes.byref(c) if c is not None else None
    need = L.lpcnet_b200_write_blob(recs, n, cp, None, 0)
    if need < 0:
        raise LPCNetB200Error("write_blob: " + _err())
    out = (ctypes.c_ubyte * need)()
    if L.lpcnet_b200_write_blob(recs, n, cp, out, need) != need:
        raise LPCNetB200Error("write_blob: " + _err())
    return bytes(out)


def blob_config(blob):
    """(gamma, delay, end2end) of the blob's lpcnet_b200_config record, or None."""
    c = Config()
    r = lib().lpcnet_b200_blob_config(blob, len(blob), ctypes.byref(c))
    if r < 0:
        raise LPCNetB200Error("blob_config: " + _err())
    return (float(c.lpc_gamma), int(c.features_delay), int(c.end2end)) if r else None


def shard_range(n, k, parts):
    a, b = ctypes.c_int(0), ctypes.c_int(0)
    if lib().lpcnet_b200_shard_range(int(n), int(k), int(parts), ctypes.byref(a), ctypes.byref(b)) != 0:
        raise LPCNetB200Error(_err())
    return int(a.value), int(a.value + b.value)


class Multi:
    """n independent streams sharded over several GPUs of ONE process (lpcnet_b200_multi_*, csrc/multi_api.cu)."""

    def __init__(self, n_streams, blob, devices, config=None, codebooks=None):
        self._L = lib()
        devs = (ctypes.c_int * len(devices))(*[int(d) for d in devices])
        c = Config(float(config[0]), int(config[1]), int(config[2])) if config is not None else None
        self._h = self._L.lpcnet_b200_multi_create(int(n_streams), blob, len(blob), ctypes.byref(c) if c is not None else None, devs, len(devices))
        if not self._h:
            raise LPCNetB200Error("lpcnet_b200_multi_create: " + _err())
        self.n = int(n_streams)
        self.devices = list(devices)
        if codebooks is not None:
            cb = np.ascontiguousarray(codebooks, dtype=np.float32)
            if self._L.lpcnet_b200_multi_set_codebooks(self._h, cb.ctypes.data, cb.size) != 0:
                raise LPCNetB200Error(_err())

    def close(self):
        if getattr(self, "_h", None):
            self._L.lpcnet_b200_multi_destroy(self._h)
            self._h = None

    __del__ = close

    def shard(self, k):
        d, a, c = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
        if self._L.lpcnet_b200_multi_shard(self._h, int(k), ctypes.byref(d), ctypes.byref(a), ctypes.byref(c)) != 0:
            raise LPCNetB200Error(_err())
        return int(d.value), int(a.value), int(c.value)

    def peer_access(self):
        return bool(self._L.lpcnet_b200_multi_peer_access(self._h))

    def reset(self):
        if self._L.lpcnet_b200_multi_reset(self._h) != 0:
            raise LPCNetB200Error(_err())

    def synthesize(self, features, samples_per_frame=160, gather=False):
        """features [n][T][stride] -> pcm [n][T*spf]; gather=True collects the PCM on devices[0] first (NVLink peer DMA) and reads it back from there."""
        f = np.ascontiguousarray(features, dtype=np.float32)
        assert f.ndim == 3 and f.shape[0] == self.n
        T, stride = f.shape[1], f.shape[2]
        pcm = np.zeros((self.n, T * samples_per_frame), dtype=np.int16)
        if not gather:
            if self._L.lpcnet_b200_multi_synthesize(self._h, f.ctypes.data, T, stride, samples_per_frame, pcm.ctypes.data) != 0:
                raise LPCNetB200Error("lpcnet_b200_multi_synthesize: " + _err())
            return pcm
        d = self._L.lpcnet_b200_device_alloc_on(self.devices[0], pcm.nbytes)
        if not d:
            raise LPCNetB200Error(_err())
        try:
            if self._L.lpcnet_b200_multi_synthesize_gather(self._h, f.ctypes.data, T, stride, samples_per_frame, d) != 0:
                raise LPCNetB200Error("lpcnet_b200_multi_synthesize_gather: " + _err())
            self._L.lpcnet_b200_set_device(self.devices[0])
            if self._L.lpcnet_b200_memcpy_d2h(pcm.ctypes.data, d, pcm.nbytes) != 0:
                raise LPCNetB200Error(_err())
        finally:
            self._L.lpcnet_b200_device_free(d)
        return pcm

    def decode(self, packets, gather=False):
        p = np.ascontiguousarray(packets, dtype=np.uint8)
        assert p.ndim == 3 and p.shape[0] == self.n and p.shape[2] == 8
        pcm = np.zeros((self.n, p.shape[1] * 640), dtype=np.int16)
        if not gather:
            if self._L.lpcnet_b200_multi_decode(self._h, p.ctypes.data, p.shape[1], pcm.ctypes.data) != 0:
                raise LPCNetB200Error("lpcnet_b200_multi_decode: " + _err())
            return pcm
        d = self._L.lpcnet_b200_device_alloc_on(self.devices[0], pcm.nbytes)
        try:
            if self._L.lpcnet_b200_multi_decode_gather(self._h, p.ctypes.data, p.shape[1], d) != 0:
                raise LPCNetB200Error("lpcnet_b200_multi_decode_gather: " + _err())
            self._L.lpcnet_b200_set_device(self.devices[0])
            self._L.lpcnet_b200_memcpy_d2h(pcm.ctypes.data, d, pcm.nbytes)
        finally:
            self._L.lpcnet_b200_device_free(d)
        return pcm


class EncBatch:
    """n independent analysis streams on one GPU (lpcnet_b200_enc_*, csrc/enc_kernels.cu): feature extraction and the encoder."""

    def __init__(self, n_streams, device=0, codebooks=None):
        self._L = lib()
        self._h = self._L.lpcnet_b200_enc_create(int(n_streams), int(device))
        if not self._h:
            raise LPCNetB200Error("lpcnet_b200_enc_create: " + _err())
        self.n = int(n_streams)
        if codebooks is not None:
            cb = np.ascontiguousarray(codebooks, dtype=np.float32)
            if self._L.lpcnet_b200_enc_set_codebooks(self._h, cb.ctypes.data, cb.size) != 0:
                raise LPCNetB200Error(_err())

    def close(self):
        if getattr(self, "_h", None):
            self._L.lpcnet_b200_enc_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self):
        if self._L.lpcnet_b200_enc_reset(self._h) != 0:
            raise LPCNetB200Error(_err())

    def reset_streams(self, streams):
        """lpcnet_encoder_init for the listed streams only (ids may repeat); the others carry on."""
        ids = np.ascontiguousarray(streams, dtype=np.int32)
        if self._L.lpcnet_b200_enc_reset_streams(self._h, ids.ctypes.data, int(ids.size)) != 0:
            raise LPCNetB200Error(_err())

    def state_size(self):
        return int(self._L.lpcnet_b200_enc_state_size(self._h))

    def export_state(self, s):
        """stream s's whole analysis state as an opaque uint8 blob of state_size() bytes"""
        buf = np.zeros(self.state_size(), dtype=np.uint8)
        if self._L.lpcnet_b200_enc_export_state(self._h, int(s), buf.ctypes.data) != 0:
            raise LPCNetB200Error(_err())
        return buf

    def import_state(self, s, buf):
        b = np.ascontiguousarray(buf).view(np.uint8).ravel()
        assert b.size == self.state_size()
        if self._L.lpcnet_b200_enc_import_state(self._h, int(s), b.ctypes.data) != 0:
            raise LPCNetB200Error(_err())

    def copy_streams(self, dst_rows, src_enc_batch, src_rows):
        """Row dst_rows[k] of this batch becomes what row src_rows[k] of src_enc_batch (this batch allowed) was before the call,
        copied on the device (lpcnet_b200_enc_copy_streams)."""
        d = np.ascontiguousarray(dst_rows, dtype=np.int32)
        s = np.ascontiguousarray(src_rows, dtype=np.int32)
        if d.shape != s.shape:
            raise LPCNetB200Error("copy_streams: %d destination rows for %d source rows" % (d.size, s.size))
        if self._L.lpcnet_b200_enc_copy_streams(self._h, d.ctypes.data, src_enc_batch._h, s.ctypes.data, int(d.size)) != 0:
            raise LPCNetB200Error("copy_streams: " + _err())

    def compute_features(self, pcm):
        """pcm [n][T*160] int16 (or float32: the _float entry point) -> features [n][T][36]."""
        p = np.ascontiguousarray(pcm)
        assert p.ndim == 2 and p.shape[0] == self.n and p.shape[1] % 160 == 0
        T = p.shape[1] // 160
        out = np.zeros((self.n, T, 36), np.float32)
        if p.dtype == np.float32:
            r = self._L.lpcnet_b200_enc_compute_features_float(self._h, p.ctypes.data, T, out.ctypes.data)
        else:
            p = np.ascontiguousarray(p, dtype=np.int16)
            r = self._L.lpcnet_b200_enc_compute_features(self._h, p.ctypes.data, T, out.ctypes.data)
        if r != 0:
            raise LPCNetB200Error("lpcnet_b200_enc_compute_features: " + _err())
        return out

    def encode(self, pcm):
        """pcm [n][P*640] int16 -> packets [n][P][8] uint8."""
        p = np.ascontiguousarray(pcm, dtype=np.int16)
        assert p.ndim == 2 and p.shape[0] == self.n and p.shape[1] % 640 == 0
        P = p.shape[1] // 640
        out = np.zeros((self.n, P, 8), np.uint8)
        if self._L.lpcnet_b200_enc_encode(self._h, p.ctypes.data, P, out.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_enc_encode: " + _err())
        return out

    def compute_features_device(self, d_pcm_ptr, nframes, d_features_ptr, cuda_stream=None):
        """d_pcm [n][nframes*160] int16 -> d_features [n][nframes][36] float32, both device pointers."""
        if self._L.lpcnet_b200_enc_compute_features_device(self._h, d_pcm_ptr, int(nframes), d_features_ptr, cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_enc_compute_features_device: " + _err())

    def encode_device(self, d_pcm_ptr, npackets, d_packets_ptr, cuda_stream=None):
        """d_pcm [n][npackets*640] int16 -> d_packets [n][npackets][8] uint8, both device pointers."""
        if self._L.lpcnet_b200_enc_encode_device(self._h, d_pcm_ptr, int(npackets), d_packets_ptr, cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_enc_encode_device: " + _err())

    def compute_features4(self, pcm):
        """pcm [n][P*640] int16 -> features [n][P*4][36] (lpcnet_compute_features: superframe analysis without quantisation)."""
        p = np.ascontiguousarray(pcm, dtype=np.int16)
        assert p.ndim == 2 and p.shape[0] == self.n and p.shape[1] % 640 == 0
        P = p.shape[1] // 640
        out = np.zeros((self.n, P * 4, 36), np.float32)
        if self._L.lpcnet_b200_enc_compute_features4(self._h, p.ctypes.data, P, out.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_enc_compute_features4: " + _err())
        return out


class Batch:
    """n independent synthesis streams stepped in lockstep on one GPU (include/lpcnet_b200.h)."""

    def __init__(self, n_streams, blob, lpc_gamma=None, device=0, codebooks=None, config=None):
        """config: (lpc_gamma, features_delay, end2end) -> lpcnet_b200_batch_create_ex; None -> lpcnet_b200_batch_create(lpc_gamma).
        lpc_gamma None: the blob's metadata record supplies it (tools/import_nnet_data.py embeds nnet_data.h's LPC_GAMMA), else 1."""
        self._L = lib()
        if config is not None:
            c = Config(float(config[0]), int(config[1]), int(config[2]))
            self._h = self._L.lpcnet_b200_batch_create_ex(int(n_streams), blob, len(blob), ctypes.byref(c), int(device))
        else:
            self._h = self._L.lpcnet_b200_batch_create(int(n_streams), blob, len(blob),
                                                        0.0 if lpc_gamma is None else float(lpc_gamma), int(device))
        if not self._h:
            raise LPCNetB200Error("lpcnet_b200_batch_create: " + _err())
        self.n = int(n_streams)
        na = ctypes.c_int(0)
        c = Config()
        self._L.lpcnet_b200_batch_model_info(self._h, ctypes.byref(na), ctypes.byref(c))
        self.na = int(na.value)
        self.config = (float(c.lpc_gamma), int(c.features_delay), int(c.end2end))
        if codebooks is not None:
            cb = np.ascontiguousarray(codebooks, dtype=np.float32)
            if self._L.lpcnet_b200_batch_set_codebooks(self._h, cb.ctypes.data, cb.size) != 0:
                raise LPCNetB200Error(_err())

    def close(self):
        if getattr(self, "_h", None):
            self._L.lpcnet_b200_batch_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self):
        if self._L.lpcnet_b200_batch_reset(self._h) != 0:
            raise LPCNetB200Error(_err())

    def synthesize(self, features, samples_per_frame=160, preload=0, pcm_in=None):
        """features [n][T][stride>=20] float32 (host) -> pcm [n][T*samples_per_frame] int16 (host).
        preload > 0 (lpcnet_synthesize_impl's teacher forcing): pcm_in [n][>=preload] supplies the forced samples."""
        f = np.ascontiguousarray(features, dtype=np.float32)
        assert f.ndim == 3 and f.shape[0] == self.n
        T, stride = f.shape[1], f.shape[2]
        pcm = np.zeros((self.n, T * samples_per_frame), dtype=np.int16)
        if preload:
            pcm[:, :preload] = np.asarray(pcm_in)[:, :preload]
        if self._L.lpcnet_b200_batch_synthesize_ex(self._h, f.ctypes.data, T, stride, samples_per_frame, pcm.ctypes.data, int(preload)) != 0:
            raise LPCNetB200Error("lpcnet_b200_batch_synthesize: " + _err())
        return pcm

    def reset_streams(self, streams):
        ids = np.ascontiguousarray(streams, dtype=np.int32)
        if self._L.lpcnet_b200_batch_reset_streams(self._h, ids.ctypes.data, int(ids.size)) != 0:
            raise LPCNetB200Error(_err())

    def reset_signal(self):
        if self._L.lpcnet_b200_batch_reset_signal(self._h) != 0:
            raise LPCNetB200Error(_err())

    def run_frame_network(self, features):
        f = np.ascontiguousarray(features, dtype=np.float32)
        if self._L.lpcnet_b200_batch_run_frame_network(self._h, f.ctypes.data, f.shape[1], f.shape[2]) != 0:
            raise LPCNetB200Error(_err())

    def synthesize_tail(self, samples, preload=0, pcm_in=None):
        pcm = np.zeros((self.n, samples), dtype=np.int16)
        if preload:
            pcm[:, :preload] = np.asarray(pcm_in)[:, :preload]
        if self._L.lpcnet_b200_batch_synthesize_tail(self._h, int(samples), pcm.ctypes.data, int(preload)) != 0:
            raise LPCNetB200Error(_err())
        return pcm

    def frame_network_deferred(self, features):
        """features [n][stride>=20]: one frame per stream queued (run_frame_network_deferred)."""
        f = np.ascontiguousarray(features, dtype=np.float32)
        if self._L.lpcnet_b200_batch_frame_network_deferred(self._h, f.ctypes.data, f.shape[1]) != 0:
            raise LPCNetB200Error(_err())

    def frame_network_flush(self):
        if self._L.lpcnet_b200_batch_frame_network_flush(self._h) != 0:
            raise LPCNetB200Error(_err())

    def export_state(self, s):
        buf = np.zeros(self._L.lpcnet_b200_batch_state_size(self._h) // 4, dtype=np.float32)
        if self._L.lpcnet_b200_batch_export_state(self._h, int(s), buf.ctypes.data) != 0:
            raise LPCNetB200Error(_err())
        return buf

    def import_state(self, s, buf):
        b = np.ascontiguousarray(buf, dtype=np.float32)
        assert b.size * 4 == self._L.lpcnet_b200_batch_state_size(self._h)
        if self._L.lpcnet_b200_batch_import_state(self._h, int(s), b.ctypes.data) != 0:
            raise LPCNetB200Error(_err())

    def snapshot(self):
        """Device-side copy of the whole batch state; returns a handle for restore()/free_snapshot()."""
        h = self._L.lpcnet_b200_batch_snapshot_create(self._h)
        if not h or self._L.lpcnet_b200_batch_snapshot_save(self._h, h) != 0:
            raise LPCNetB200Error(_err())
        return h

    def restore(self, snap):
        if self._L.lpcnet_b200_batch_snapshot_restore(self._h, snap) != 0:
            raise LPCNetB200Error(_err())

    def free_snapshot(self, snap):
        self._L.lpcnet_b200_batch_snapshot_destroy(snap)

    def copy_streams(self, dst_rows, src_batch, src_rows):
        """Row dst_rows[k] of this batch becomes what row src_rows[k] of src_batch (this batch allowed) was before the call: the whole
        stream state, its deferred frames and its tail conditioning, copied on the device (lpcnet_b200_batch_copy_streams)."""
        d = np.ascontiguousarray(dst_rows, dtype=np.int32)
        s = np.ascontiguousarray(src_rows, dtype=np.int32)
        if d.shape != s.shape:
            raise LPCNetB200Error("copy_streams: %d destination rows for %d source rows" % (d.size, s.size))
        if self._L.lpcnet_b200_batch_copy_streams(self._h, d.ctypes.data, src_batch._h, s.ctypes.data, int(d.size)) != 0:
            raise LPCNetB200Error("copy_streams: " + _err())

    def set_pcm_sink(self, d_ptr, pitch_samples, first_row):
        if self._L.lpcnet_b200_batch_set_pcm_sink(self._h, d_ptr, int(pitch_samples), int(first_row)) != 0:
            raise LPCNetB200Error(_err())

    def synthesize_device(self, d_features_ptr, nframes, stride, d_pcm_ptr, samples_per_frame=160, cuda_stream=None, preload=0):
        """Device pointers in and out.  preload > 0: the first `preload` samples of every stream's row of d_pcm hold the forced
        signal of the first frame (lpcnet_b200_batch_synthesize_device_ex)."""
        if preload:
            r = self._L.lpcnet_b200_batch_synthesize_device_ex(self._h, d_features_ptr, nframes, stride, samples_per_frame, d_pcm_ptr, int(preload), cuda_stream)
        else:
            r = self._L.lpcnet_b200_batch_synthesize_device(self._h, d_features_ptr, nframes, stride, samples_per_frame, d_pcm_ptr, cuda_stream)
        if r != 0:
            raise LPCNetB200Error("lpcnet_b200_batch_synthesize_device: " + _err())

    def decode(self, packets):
        """packets [n][P][8] uint8 -> pcm [n][P*640] int16."""
        p = np.ascontiguousarray(packets, dtype=np.uint8)
        assert p.ndim == 3 and p.shape[0] == self.n and p.shape[2] == 8
        pcm = np.empty((self.n, p.shape[1] * 640), dtype=np.int16)
        if self._L.lpcnet_b200_batch_decode(self._h, p.ctypes.data, p.shape[1], pcm.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_batch_decode: " + _err())
        return pcm

    def decode_device(self, d_packets_ptr, npackets, d_pcm_ptr, cuda_stream=None):
        if self._L.lpcnet_b200_batch_decode_device(self._h, d_packets_ptr, npackets, d_pcm_ptr, cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_batch_decode_device: " + _err())

    def timer_start(self):
        if self._L.lpcnet_b200_batch_timer_start(self._h) != 0:
            raise LPCNetB200Error(_err())

    def timer_stop(self):
        ms = self._L.lpcnet_b200_batch_timer_stop(self._h)
        if ms < 0:
            raise LPCNetB200Error(_err())
        return float(ms)

    def flush_l2(self):
        if self._L.lpcnet_b200_batch_flush_l2(self._h) != 0:
            raise LPCNetB200Error(_err())

    def sync(self):
        if self._L.lpcnet_b200_batch_sync(self._h) != 0:
            raise LPCNetB200Error(_err())

    def last_sample_kernel_ms(self):
        k = ctypes.c_int(0)
        ms = self._L.lpcnet_b200_batch_last_sample_kernel_ms(self._h, ctypes.byref(k))
        return float(ms), int(k.value)

    def algorithmic_bytes(self):
        a, b = ctypes.c_long(0), ctypes.c_long(0)
        self._L.lpcnet_b200_batch_algorithmic_bytes(self._h, ctypes.byref(a), ctypes.byref(b))
        return int(a.value), int(b.value)

    def get_state(self, s):
        ga = np.zeros(self.na, np.float32); gb = np.zeros(16, np.float32); ls = np.zeros(16, np.float32)
        misc = np.zeros(2, np.int32); rng = np.zeros(4, np.uint32)
        if self._L.lpcnet_b200_batch_get_state(self._h, int(s), ga.ctypes.data, gb.ctypes.data, ls.ctypes.data, misc.ctypes.data, rng.ctypes.data) != 0:
            raise LPCNetB200Error(_err())
        return dict(gru_a=ga, gru_b=gb, last_sig=ls, last_exc=int(misc[0]), frame_count=int(misc[1]), rng=rng)

    def debug_frame_network(self, features):
        f = np.ascontiguousarray(features, dtype=np.float32)
        T, stride = f.shape[1], f.shape[2]
        ga = np.zeros((self.n, T, 3 * self.na), np.float32); gb = np.zeros((self.n, T, 48), np.float32); lpc = np.zeros((self.n, T, 16), np.float32)
        if self._L.lpcnet_b200_debug_frame_network(self._h, f.ctypes.data, T, stride, ga.ctypes.data, gb.ctypes.data, lpc.ctypes.data) != 0:
            raise LPCNetB200Error(_err())
        return ga, gb, lpc

    def debug_rcp(self, x):
        """The engine's _mm256_rcp_ps emulation (the per-sample kernels' table) for an array of floats."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        a = np.zeros_like(x)
        if self._L.lpcnet_b200_debug_rcp(self._h, x.ctypes.data, a.ctypes.data, int(x.size)) != 0:
            raise LPCNetB200Error(_err())
        return a

    def debug_tanh_x86(self, x):
        """(rcp, tanh) of the conditioning network's full-range activation for an array of floats."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        a = np.zeros_like(x); b = np.zeros_like(x)
        if self._L.lpcnet_b200_debug_tanh_x86(self._h, x.ctypes.data, a.ctypes.data, b.ctypes.data, int(x.size)) != 0:
            raise LPCNetB200Error(_err())
        return a, b


def group_plan(sizes, sms, override_spc=0):
    """Launch plan of a group whose members have `sizes` streams on `sms` SMs: (streams per CTA, CTA count)
    (lpcnet_b200_debug_group_plan; host only, needs no GPU)."""
    n = (ctypes.c_int * len(sizes))(*[int(v) for v in sizes])
    spc, ctas = ctypes.c_int(0), ctypes.c_int(0)
    if lib().lpcnet_b200_debug_group_plan(n, len(sizes), int(sms), int(override_spc), ctypes.byref(spc), ctypes.byref(ctas)) != 0:
        raise LPCNetB200Error("debug_group_plan: " + _err())
    return int(spc.value), int(ctas.value)


def group_plan_float(sizes, sms, override_spc=0, lane_stream=False):
    """Launch plan of a float group whose members have `sizes` streams on `sms` SMs: (kernel, streams per CTA, slots, CTA count),
    kernel "neuron" (neuron-per-lane, `slots` = 1, 2 or 4 streams per CTA) or "lane" (lane == stream, slots = spc);
    lane_stream stands for LPCNET_B200_FLOAT_LANE_STREAM (lpcnet_b200_debug_group_plan_float; host only, needs no GPU)."""
    n = (ctypes.c_int * len(sizes))(*[int(v) for v in sizes])
    spc, slots, ctas = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    r = lib().lpcnet_b200_debug_group_plan_float(n, len(sizes), int(sms), int(override_spc), int(bool(lane_stream)),
                                                 ctypes.byref(spc), ctypes.byref(slots), ctypes.byref(ctas))
    if r < 0:
        raise LPCNetB200Error("debug_group_plan_float: " + _err())
    return ("neuron" if r == 1 else "lane"), int(spc.value), int(slots.value), int(ctas.value)


def mixed_plan(sizes, na, is_float, sms, override_spc=0, lane_stream=False):
    """Launch plan of a mixed group whose member k has sizes[k] streams, na[k] GRU_A units and flavour is_float[k] on `sms` SMs:
    (streams per CTA, class of each member, [(kernel, CTA count) per class]) with kernel "int8", "neuron" or "lane" (the float
    kernels of group_plan_float); lane_stream stands for LPCNET_B200_FLOAT_LANE_STREAM (lpcnet_b200_debug_mixed_plan; host only,
    needs no GPU)."""
    k = len(sizes)
    if len(na) != k or len(is_float) != k:
        raise LPCNetB200Error("mixed_plan: sizes, na and is_float differ in length")
    arr = lambda v: (ctypes.c_int * max(k, 1))(*[int(x) for x in v])
    cls, ctas, neuron = arr([0] * k), arr([0] * k), arr([0] * k)
    spc = ctypes.c_int(0)
    r = lib().lpcnet_b200_debug_mixed_plan(arr(sizes), arr(na), arr(is_float), k, int(sms), int(override_spc), int(bool(lane_stream)),
                                           ctypes.byref(spc), cls, ctas, neuron)
    if r < 0:
        raise LPCNetB200Error("debug_mixed_plan: " + _err())
    first = {int(cls[j]): j for j in reversed(range(k))}          # a member of each class
    kernels = [("neuron" if neuron[c] else "lane") if is_float[first[c]] else "int8" for c in range(r)]
    return int(spc.value), [int(cls[j]) for j in range(k)], [(kernels[c], int(ctas[c])) for c in range(r)]


class Group:
    """The synthesize / decode calls of several Batch objects of one flavour (all int8 or all float) and one GRU_A size on one
    device as one call: one per-sample launch for all their streams (lpcnet_b200_group_*).  Group stream rows = batches[0]'s
    streams, then batches[1]'s, ...
    The members stay usable on their own; the group keeps them alive and must be closed before they are."""

    def __init__(self, batches):
        self._L = lib()
        self.batches = list(batches)
        hs = (c_p * len(self.batches))(*[b._h for b in self.batches])
        self._h = self._L.lpcnet_b200_group_create(hs, len(self.batches))
        if not self._h:
            raise LPCNetB200Error("lpcnet_b200_group_create: " + _err())
        self.n = int(self._L.lpcnet_b200_group_streams(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._L.lpcnet_b200_group_destroy(self._h)
            self._h = None

    __del__ = close

    def synthesize(self, features, samples_per_frame=160):
        """features [sum n][T][stride>=20] float32 (host) -> pcm [sum n][T*samples_per_frame] int16 (host)."""
        f = np.ascontiguousarray(features, dtype=np.float32)
        assert f.ndim == 3 and f.shape[0] == self.n
        T, stride = f.shape[1], f.shape[2]
        pcm = np.zeros((self.n, T * samples_per_frame), dtype=np.int16)
        if self._L.lpcnet_b200_group_synthesize(self._h, f.ctypes.data, T, stride, samples_per_frame, pcm.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_group_synthesize: " + _err())
        return pcm

    def synthesize_device(self, d_features_ptr, nframes, stride, d_pcm_ptr, samples_per_frame=160, cuda_stream=None):
        if self._L.lpcnet_b200_group_synthesize_device(self._h, d_features_ptr, nframes, stride, samples_per_frame, d_pcm_ptr, cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_group_synthesize_device: " + _err())

    def decode(self, packets):
        """packets [sum n][P][8] uint8 -> pcm [sum n][P*640] int16."""
        p = np.ascontiguousarray(packets, dtype=np.uint8)
        assert p.ndim == 3 and p.shape[0] == self.n and p.shape[2] == 8
        pcm = np.empty((self.n, p.shape[1] * 640), dtype=np.int16)
        if self._L.lpcnet_b200_group_decode(self._h, p.ctypes.data, p.shape[1], pcm.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_group_decode: " + _err())
        return pcm

    def decode_device(self, d_packets_ptr, npackets, d_pcm_ptr, cuda_stream=None):
        if self._L.lpcnet_b200_group_decode_device(self._h, d_packets_ptr, npackets, d_pcm_ptr, cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_group_decode_device: " + _err())

    def last_sample_kernel_ms(self):
        k = ctypes.c_int(0)
        ms = self._L.lpcnet_b200_group_last_sample_kernel_ms(self._h, ctypes.byref(k))
        return float(ms), int(k.value)


class _OwnedGroup(Group):
    """a group another object holds (MultiGroup.group): the same calls, but closing it leaves the group alone"""

    def __init__(self, h, owner):
        self._L = lib()
        self._h, self._owner, self.batches = h, owner, None
        self.n = int(self._L.lpcnet_b200_group_streams(h))

    def close(self):
        self._h = None

    __del__ = close


class MultiGroup:
    """Several Multi objects, one per model, all over the same devices and of one flavour and GRU_A size, served by one call: on
    every device one group over the members' shards (lpcnet_b200_multi_group_*).  Rows = multis[0]'s streams, then multis[1]'s, ...
    The members stay usable on their own; the multi-group keeps them alive and must be closed before they are."""

    def __init__(self, multis):
        self._L = lib()
        self.multis = list(multis)
        hs = (c_p * len(self.multis))(*[m._h for m in self.multis])
        self._h = self._L.lpcnet_b200_multi_group_create(hs, len(self.multis))
        if not self._h:
            raise LPCNetB200Error("lpcnet_b200_multi_group_create: " + _err())
        self.n = int(self._L.lpcnet_b200_multi_group_streams(self._h))
        self.devices = list(self.multis[0].devices)

    def close(self):
        if getattr(self, "_h", None):
            self._L.lpcnet_b200_multi_group_destroy(self._h)
            self._h = None

    __del__ = close

    def group(self, k):
        """the group of devices[k] (last_sample_kernel_ms of its part of the last call)"""
        h = self._L.lpcnet_b200_multi_group_group(self._h, int(k))
        if not h:
            raise LPCNetB200Error(_err())
        return _OwnedGroup(h, self)

    def _gathered(self, call, pcm):
        d = self._L.lpcnet_b200_device_alloc_on(self.devices[0], pcm.nbytes)
        if not d:
            raise LPCNetB200Error(_err())
        try:
            call(d)
            self._L.lpcnet_b200_set_device(self.devices[0])
            if self._L.lpcnet_b200_memcpy_d2h(pcm.ctypes.data, d, pcm.nbytes) != 0:
                raise LPCNetB200Error(_err())
        finally:
            self._L.lpcnet_b200_device_free(d)
        return pcm

    def synthesize(self, features, samples_per_frame=160, gather=False):
        """features [sum n][T][stride>=20] -> pcm [sum n][T*spf]; gather=True collects the PCM on devices[0] first and reads it back
        from there."""
        f = np.ascontiguousarray(features, dtype=np.float32)
        if f.ndim != 3 or f.shape[0] != self.n:
            raise LPCNetB200Error("multi_group synthesize: features of shape %s for %d streams" % (f.shape, self.n))
        T, stride = f.shape[1], f.shape[2]
        pcm = np.zeros((self.n, T * samples_per_frame), dtype=np.int16)

        def call(d):
            fn = self._L.lpcnet_b200_multi_group_synthesize_gather if d else self._L.lpcnet_b200_multi_group_synthesize
            if fn(self._h, f.ctypes.data, T, stride, samples_per_frame, d or pcm.ctypes.data) != 0:
                raise LPCNetB200Error("lpcnet_b200_multi_group_synthesize%s: %s" % ("_gather" if d else "", _err()))
        if gather:
            return self._gathered(call, pcm)
        call(None)
        return pcm

    def decode(self, packets, gather=False):
        """packets [sum n][P][8] uint8 -> pcm [sum n][P*640] int16."""
        p = np.ascontiguousarray(packets, dtype=np.uint8)
        if p.ndim != 3 or p.shape[0] != self.n or p.shape[2] != 8:
            raise LPCNetB200Error("multi_group decode: packets of shape %s for %d streams" % (p.shape, self.n))
        pcm = np.zeros((self.n, p.shape[1] * 640), dtype=np.int16)

        def call(d):
            fn = self._L.lpcnet_b200_multi_group_decode_gather if d else self._L.lpcnet_b200_multi_group_decode
            if fn(self._h, p.ctypes.data, p.shape[1], d or pcm.ctypes.data) != 0:
                raise LPCNetB200Error("lpcnet_b200_multi_group_decode%s: %s" % ("_gather" if d else "", _err()))
        if gather:
            return self._gathered(call, pcm)
        call(None)
        return pcm


class MixedGroup:
    """Batch objects of any GRU_A sizes and flavours on one device served by one call: one group per (GRU_A size, flavour) class,
    all planned together so that they fit on the SMs at once, each class's launches on a CUDA stream of its own
    (lpcnet_b200_mixed_group_*).  Rows = batches[0]'s streams, then batches[1]'s, ...
    The members stay usable on their own; the mixed group keeps them alive and must be closed before they are."""

    def __init__(self, batches):
        self._L = lib()
        self.batches = list(batches)
        hs = (c_p * max(len(self.batches), 1))(*[b._h if b is not None else None for b in self.batches])
        self._h = self._L.lpcnet_b200_mixed_group_create(hs if self.batches else None, len(self.batches))
        if not self._h:
            raise LPCNetB200Error("lpcnet_b200_mixed_group_create: " + _err())
        self.n = int(self._L.lpcnet_b200_mixed_group_streams(self._h))
        self.classes = int(self._L.lpcnet_b200_mixed_group_classes(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._L.lpcnet_b200_mixed_group_destroy(self._h)
            self._h = None

    __del__ = close

    def group(self, c):
        """class c's group (last_sample_kernel_ms of its part of the last call)"""
        h = self._L.lpcnet_b200_mixed_group_group(self._h, int(c))
        if not h:
            raise LPCNetB200Error(_err())
        return _OwnedGroup(h, self)

    def synthesize(self, features, samples_per_frame=160):
        """features [sum n][T][stride>=20] float32 (host) -> pcm [sum n][T*samples_per_frame] int16 (host)."""
        f = np.ascontiguousarray(features, dtype=np.float32)
        if f.ndim != 3 or f.shape[0] != self.n:
            raise LPCNetB200Error("mixed_group synthesize: features of shape %s for %d streams" % (f.shape, self.n))
        T, stride = f.shape[1], f.shape[2]
        pcm = np.zeros((self.n, T * samples_per_frame), dtype=np.int16)
        if self._L.lpcnet_b200_mixed_group_synthesize(self._h, f.ctypes.data, T, stride, samples_per_frame, pcm.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_mixed_group_synthesize: " + _err())
        return pcm

    def synthesize_device(self, d_features_ptr, nframes, stride, d_pcm_ptr, samples_per_frame=160, cuda_stream=None):
        if self._L.lpcnet_b200_mixed_group_synthesize_device(self._h, d_features_ptr, nframes, stride, samples_per_frame, d_pcm_ptr,
                                                             cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_mixed_group_synthesize_device: " + _err())

    def decode(self, packets):
        """packets [sum n][P][8] uint8 -> pcm [sum n][P*640] int16."""
        p = np.ascontiguousarray(packets, dtype=np.uint8)
        if p.ndim != 3 or p.shape[0] != self.n or p.shape[2] != 8:
            raise LPCNetB200Error("mixed_group decode: packets of shape %s for %d streams" % (p.shape, self.n))
        pcm = np.zeros((self.n, p.shape[1] * 640), dtype=np.int16)
        if self._L.lpcnet_b200_mixed_group_decode(self._h, p.ctypes.data, p.shape[1], pcm.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_b200_mixed_group_decode: " + _err())
        return pcm

    def decode_device(self, d_packets_ptr, npackets, d_pcm_ptr, cuda_stream=None):
        if self._L.lpcnet_b200_mixed_group_decode_device(self._h, d_packets_ptr, npackets, d_pcm_ptr, cuda_stream) != 0:
            raise LPCNetB200Error("lpcnet_b200_mixed_group_decode_device: " + _err())

    def last_call_ms(self):
        """device time of the last call, fork to join"""
        return float(self._L.lpcnet_b200_mixed_group_last_call_ms(self._h))


class LPCNet:
    """Mirror of the reference single-stream API: lpcnet_create / lpcnet_load_model / lpcnet_synthesize / lpcnet_reset."""

    def __init__(self, blob=None):
        self._L = lib()
        self._st = self._L.lpcnet_create()
        if not self._st:
            raise LPCNetB200Error("lpcnet_create: " + _err())
        if blob is not None:
            self.load_model(blob)

    def load_model(self, blob):
        if self._L.lpcnet_load_model(self._st, blob, len(blob)) != 0:
            raise LPCNetB200Error("lpcnet_load_model: " + _err())

    def reset(self):
        self._L.lpcnet_reset(self._st)

    def synthesize(self, features, N=160):
        f = np.ascontiguousarray(features, dtype=np.float32)
        out = np.zeros(N, dtype=np.int16)
        self._L.lpcnet_synthesize(self._st, f.ctypes.data, out.ctypes.data, N)
        return out

    def close(self):
        if getattr(self, "_st", None):
            self._L.lpcnet_destroy(self._st)
            self._st = None

    __del__ = close


class LPCNetDecoder:
    """Mirror of lpcnet_decoder_create / lpcnet_decode (model is loaded through the leading LPCNetState member)."""

    def __init__(self, blob=None):
        self._L = lib()
        self._st = self._L.lpcnet_decoder_create()
        if not self._st:
            raise LPCNetB200Error("lpcnet_decoder_create: " + _err())
        if blob is not None and self._L.lpcnet_load_model(self._st, blob, len(blob)) != 0:
            raise LPCNetB200Error("lpcnet_load_model: " + _err())

    def decode(self, packet):
        p = np.ascontiguousarray(packet, dtype=np.uint8)
        out = np.zeros(640, dtype=np.int16)
        if self._L.lpcnet_decode(self._st, p.ctypes.data, out.ctypes.data) != 0:
            raise LPCNetB200Error("lpcnet_decode: " + _err())
        return out

    def close(self):
        if getattr(self, "_st", None):
            self._L.lpcnet_decoder_destroy(self._st)
            self._st = None

    __del__ = close
