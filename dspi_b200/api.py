"""ctypes binding of the C ABI (``include/dspi_b200.h``) — the call a Python host makes.

There is no CPU path in this package: if ``libdspi_b200.so`` is missing or no
sm_90 device is visible, construction fails loudly.
"""
import ctypes as C
import os

import numpy as np

from . import layouts as L

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libdspi_b200.so")

ARITH_F32_FUSED, ARITH_F32_STRICT, ARITH_Q28 = 0, 1, 2
ARITH = {"f32f": ARITH_F32_FUSED, "f32s": ARITH_F32_STRICT, "q28": ARITH_Q28}

# every symbol include/dspi_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    "dspi_last_error", "dspi_device_count", "dspi_compute_coefficients_f32", "dspi_compute_coefficients_q28",
    "dspi_eq_create", "dspi_eq_destroy", "dspi_eq_upload_biquads", "dspi_eq_download_biquads", "dspi_eq_set_param",
    "dspi_eq_process_device", "dspi_eq_process_host", "dspi_eq_sync", "dspi_eq_stream", "dspi_eq_launch_count",
    "dspi_eq_kernel_info", "dspi_eq_set_params_device", "dspi_chain_set_eq_params_device", "dspi_chainq_set_eq_params_device",
    "dspi_chain_state_size", "dspi_chain_state_export", "dspi_chain_state_import", "dspi_chainq_state_size", "dspi_chainq_state_export", "dspi_chainq_state_import",
    "dspi_host_alloc", "dspi_host_free",
    "dspi_chain_create", "dspi_chain_destroy", "dspi_chain_set_params", "dspi_chain_upload_biquads", "dspi_chain_download_biquads",
    "dspi_chain_reset_state", "dspi_chain_process_host", "dspi_chain_process_device", "dspi_chain_sync", "dspi_chain_stream",
    "dspi_chain_launch_count", "dspi_delay_samples",
    "dspi_crossfeed_compute_coefficients_f32", "dspi_leveller_compute_coefficients", "dspi_loudness_compute_table_f32", "dspi_host_volume",
    "dspi_chainq_create", "dspi_chainq_destroy", "dspi_chainq_set_params", "dspi_chainq_upload_biquads", "dspi_chainq_download_biquads",
    "dspi_chainq_reset_state", "dspi_chainq_process_host", "dspi_chainq_process_device", "dspi_chainq_sync", "dspi_chainq_launch_count",
    "dspi_crossfeed_compute_coefficients_q28", "dspi_loudness_compute_table_q28",
    "dspi_spdif_lookup_table", "dspi_spdif_encode_device", "dspi_spdif_encode_host",
    "dspi_bulk_state_defaults", "dspi_bulk_params_apply", "dspi_bulk_params_collect", "dspi_bulk_state_to_chain_f32", "dspi_bulk_state_to_chain_q28",
    "dspi_preset_slot_size", "dspi_crc32", "dspi_preset_slot_apply", "dspi_preset_slot_collect",
    "dspi_preamp", "dspi_master_volume", "dspi_preset_mute_arm", "dspi_preset_mute_step",
    "dspi_nccl_unique_id", "dspi_sg_create", "dspi_sg_destroy", "dspi_sg_process",
    "dspi_chainq_stream", "dspi_eq_process_device_range", "dspi_bind_host_to_device", "dspi_eqx_create", "dspi_eqx_destroy", "dspi_eqx_shard_range",
    "dspi_eqx_upload_biquads", "dspi_eqx_download_biquads", "dspi_eqx_process_host", "dspi_eqx_process_root", "dspi_eqx_launch_count",
    "dspi_chain_set_dynamics_device", "dspi_chainq_set_dynamics_device", "dspi_chain_sm_partition", "dspi_chainq_sm_partition",
    "dspi_chain_set_preset_mute", "dspi_chain_get_preset_mute", "dspi_chainq_set_preset_mute", "dspi_chainq_get_preset_mute",
    "dspi_chain_process_packets_host", "dspi_chain_process_packets_device", "dspi_chainq_process_packets_host", "dspi_chainq_process_packets_device",
    "dspi_chain_set_spdif_tx", "dspi_chain_get_spdif_tx", "dspi_chainq_set_spdif_tx", "dspi_chainq_get_spdif_tx",
    "dspi_chain_process_subframes_host", "dspi_chain_process_subframes_device", "dspi_chainq_process_subframes_host", "dspi_chainq_process_subframes_device",
    "dspi_eq_response_host", "dspi_eq_response_device", "dspi_chain_response_host", "dspi_chain_response_device",
    "dspi_chainq_response_host", "dspi_chainq_response_device",
    "dspi_chain_apply_bulk_device", "dspi_chainq_apply_bulk_device",
    "dspi_chain_collect_bulk_device", "dspi_chainq_collect_bulk_device",
    "dspi_chain_set_rate_device", "dspi_chainq_set_rate_device",
    "dspi_chain_edit_bulk_device", "dspi_chainq_edit_bulk_device",
    "dspi_chain_apply_preset_device", "dspi_chainq_apply_preset_device",
    "dspi_chain_collect_preset_device", "dspi_chainq_collect_preset_device",
    "dspi_chain_instance_image_size", "dspi_chain_export_instances", "dspi_chain_import_instances", "dspi_chain_reset_instances",
    "dspi_chainq_instance_image_size", "dspi_chainq_export_instances", "dspi_chainq_import_instances", "dspi_chainq_reset_instances",
    "dspi_chain_copy_instances", "dspi_chainq_copy_instances",
    "dspi_chain_process_packets_range_host", "dspi_chain_process_packets_range_device",
    "dspi_chain_process_subframes_range_host", "dspi_chain_process_subframes_range_device",
    "dspi_chainq_process_packets_range_host", "dspi_chainq_process_packets_range_device",
    "dspi_chainq_process_subframes_range_host", "dspi_chainq_process_subframes_range_device",
    "dspi_chain_lane_open", "dspi_chain_lane_close", "dspi_chain_lane_process_packets_device", "dspi_chain_lane_process_subframes_device",
    "dspi_chain_lane_stream", "dspi_chain_lane_sync",
    "dspi_chainq_lane_open", "dspi_chainq_lane_close", "dspi_chainq_lane_process_packets_device", "dspi_chainq_lane_process_subframes_device",
    "dspi_chainq_lane_stream", "dspi_chainq_lane_sync",
    "dspi_chain_lane_edit_bulk_device", "dspi_chain_lane_set_preset_mute", "dspi_chain_lane_set_spdif_tx", "dspi_chain_lane_reset_instances",
    "dspi_chainq_lane_edit_bulk_device", "dspi_chainq_lane_set_preset_mute", "dspi_chainq_lane_set_spdif_tx", "dspi_chainq_lane_reset_instances",
    "dspi_chain_lane_apply_bulk_device", "dspi_chain_lane_apply_preset_device", "dspi_chain_lane_set_rate_device",
    "dspi_chainq_lane_apply_bulk_device", "dspi_chainq_lane_apply_preset_device", "dspi_chainq_lane_set_rate_device",
    "dspi_chain_lane_collect_bulk_device", "dspi_chain_lane_collect_preset_device", "dspi_chain_lane_export_instances",
    "dspi_chain_lane_response_device", "dspi_chain_lane_get_preset_mute", "dspi_chain_lane_get_spdif_tx",
    "dspi_chainq_lane_collect_bulk_device", "dspi_chainq_lane_collect_preset_device", "dspi_chainq_lane_export_instances",
    "dspi_chainq_lane_response_device", "dspi_chainq_lane_get_preset_mute", "dspi_chainq_lane_get_spdif_tx",
    "dspi_chain_lane_import_instances", "dspi_chain_lane_copy_instances", "dspi_chainq_lane_import_instances", "dspi_chainq_lane_copy_instances",
    "dspi_chain_lane_process_packets_host", "dspi_chain_lane_process_subframes_host",
    "dspi_chainq_lane_process_packets_host", "dspi_chainq_lane_process_subframes_host",
]


class DspiError(RuntimeError):
    pass


class _ChainDesc(C.Structure):
    _fields_ = [("arith", C.c_uint32), ("n_instances", C.c_uint32), ("n_bands", C.c_uint32),
                ("device", C.c_int32), ("max_frames", C.c_uint32)]


class _EqDesc(C.Structure):
    _fields_ = [("arith", C.c_uint32), ("n_channels", C.c_uint32), ("n_bands", C.c_uint32),
                ("device", C.c_int32), ("flags", C.c_uint32)]


_lib = None


class _EqxDesc(C.Structure):
    _fields_ = [("arith", C.c_uint32), ("n_channels", C.c_uint32), ("n_bands", C.c_uint32), ("n_devices", C.c_uint32),
                ("devices", C.c_int32 * 8), ("flags", C.c_uint32)]


def lib():
    """The loaded shared library (never built implicitly here: see ``dspi_b200.build``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DspiError(f"{LIB_PATH} is missing - build it with `python -m dspi_b200.build` "
                            "(there is no CPU fallback)")
        h = C.CDLL(LIB_PATH)
        vp, u32 = C.c_void_p, C.c_uint32
        h.dspi_last_error.restype = C.c_char_p
        h.dspi_device_count.restype = C.c_int
        h.dspi_compute_coefficients_f32.argtypes = [vp, vp, C.c_float]
        h.dspi_compute_coefficients_q28.argtypes = [vp, vp, C.c_float]
        h.dspi_eq_create.argtypes = [C.POINTER(vp), C.POINTER(_EqDesc)]
        h.dspi_eq_destroy.argtypes = [vp]
        h.dspi_eq_upload_biquads.argtypes = [vp, u32, u32, vp]
        h.dspi_eq_download_biquads.argtypes = [vp, u32, u32, vp]
        h.dspi_eq_set_param.argtypes = [vp, u32, vp, C.c_float]
        h.dspi_eq_process_device.argtypes = [vp, vp, u32, u32]
        h.dspi_eq_process_host.argtypes = [vp, vp, u32]
        h.dspi_eq_sync.argtypes = [vp]
        h.dspi_eq_stream.argtypes = [vp]
        h.dspi_eq_stream.restype = vp
        h.dspi_eq_launch_count.argtypes = [vp]
        h.dspi_eq_launch_count.restype = C.c_uint64
        h.dspi_eq_kernel_info.argtypes = [vp, C.c_char_p, C.c_size_t]
        h.dspi_delay_samples.argtypes = [C.c_float, C.c_float, C.c_int]
        h.dspi_delay_samples.restype = C.c_int32
        h.dspi_crossfeed_compute_coefficients_q28.argtypes = [vp, vp, C.c_float]
        h.dspi_loudness_compute_table_q28.argtypes = [vp, C.c_float, C.c_float, C.c_float]
        h.dspi_crossfeed_compute_coefficients_f32.argtypes = [vp, vp, C.c_float]
        h.dspi_leveller_compute_coefficients.argtypes = [vp, vp, C.c_float]
        h.dspi_loudness_compute_table_f32.argtypes = [vp, C.c_float, C.c_float, C.c_float]
        h.dspi_host_volume.argtypes = [C.c_int16, vp]
        h.dspi_host_volume.restype = C.c_int16
        h.dspi_preamp.argtypes = [C.c_float, vp, vp]
        h.dspi_master_volume.argtypes = [C.c_float, vp, vp]
        h.dspi_preset_mute_arm.argtypes = [vp, u32]
        h.dspi_preset_mute_step.argtypes = [vp, u32, u32]
        h.dspi_preset_mute_step.restype = C.c_float
        for pre in ("dspi_chain", "dspi_chainq"):
            getattr(h, pre + "_create").argtypes = [C.POINTER(vp), C.POINTER(_ChainDesc)]
            getattr(h, pre + "_destroy").argtypes = [vp]
            getattr(h, pre + "_set_params").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_upload_biquads").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_download_biquads").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_reset_state").argtypes = [vp]
            getattr(h, pre + "_process_host").argtypes = [vp, vp, u32, u32, u32, vp, vp, vp]
            getattr(h, pre + "_process_device").argtypes = [vp, vp, u32, u32, u32, vp, vp, vp]
            getattr(h, pre + "_sync").argtypes = [vp]
            getattr(h, pre + "_stream").argtypes = [vp]
            getattr(h, pre + "_stream").restype = vp
            getattr(h, pre + "_launch_count").argtypes = [vp]
            getattr(h, pre + "_launch_count").restype = C.c_uint64
            getattr(h, pre + "_state_size").argtypes = [vp]
            getattr(h, pre + "_state_size").restype = C.c_size_t
            getattr(h, pre + "_instance_image_size").argtypes = [vp]
            getattr(h, pre + "_instance_image_size").restype = C.c_size_t
            getattr(h, pre + "_export_instances").argtypes = [vp, u32, u32, vp, C.c_size_t]
            getattr(h, pre + "_import_instances").argtypes = [vp, u32, u32, vp, C.c_size_t]
            getattr(h, pre + "_reset_instances").argtypes = [vp, u32, u32]
            getattr(h, pre + "_copy_instances").argtypes = [vp, u32, vp, vp]
            getattr(h, pre + "_set_preset_mute").argtypes = [vp, u32, u32, vp, u32]
            getattr(h, pre + "_get_preset_mute").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_set_dynamics_device").argtypes = [vp, u32, u32, vp, C.c_float]
            getattr(h, pre + "_sm_partition").argtypes = [vp, vp, vp]
            getattr(h, pre + "_apply_bulk_device").argtypes = [vp, u32, u32, vp, vp, C.c_int, C.c_float, vp]
            getattr(h, pre + "_collect_bulk_device").argtypes = [vp, u32, u32, vp, vp, vp]
            getattr(h, pre + "_set_rate_device").argtypes = [vp, u32, u32, vp, vp]
            getattr(h, pre + "_edit_bulk_device").argtypes = [vp, u32, vp, C.c_int, C.c_float, vp]
            getattr(h, pre + "_apply_preset_device").argtypes = [vp, u32, u32, vp, C.c_size_t, vp, vp, C.c_float, vp]
            getattr(h, pre + "_collect_preset_device").argtypes = [vp, u32, u32, vp, vp, C.c_size_t, vp]
            getattr(h, pre + "_process_packets_host").argtypes = [vp, vp, u32, u32, vp, vp, vp, vp]
            getattr(h, pre + "_process_packets_device").argtypes = [vp, vp, u32, u32, vp, vp, vp, vp]
            getattr(h, pre + "_set_spdif_tx").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_get_spdif_tx").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_process_subframes_host").argtypes = [vp, vp, u32, u32, vp, vp, vp, vp]
            getattr(h, pre + "_process_subframes_device").argtypes = [vp, vp, u32, u32, vp, vp, vp, vp]
            for form in ("packets", "subframes"):
                for where in ("host", "device"):
                    getattr(h, "%s_process_%s_range_%s" % (pre, form, where)).argtypes = [vp, u32, u32, vp, u32, u32, vp, vp, vp, vp]
                for where in ("device", "host"):
                    getattr(h, "%s_lane_process_%s_%s" % (pre, form, where)).argtypes = [vp, u32, u32, u32, vp, u32, u32, vp, vp, vp, vp]
            getattr(h, pre + "_lane_open").argtypes = [vp, u32, u32, vp]
            getattr(h, pre + "_lane_close").argtypes = [vp, u32]
            getattr(h, pre + "_lane_stream").argtypes = [vp, u32]
            getattr(h, pre + "_lane_stream").restype = vp
            getattr(h, pre + "_lane_sync").argtypes = [vp, u32]
            getattr(h, pre + "_lane_edit_bulk_device").argtypes = [vp, u32, u32, vp, C.c_int, C.c_float, vp]
            getattr(h, pre + "_lane_set_preset_mute").argtypes = [vp, u32, u32, u32, vp, u32]
            getattr(h, pre + "_lane_set_spdif_tx").argtypes = [vp, u32, u32, u32, vp]
            getattr(h, pre + "_lane_reset_instances").argtypes = [vp, u32, u32, u32]
            getattr(h, pre + "_lane_apply_bulk_device").argtypes = [vp, u32, u32, u32, vp, vp, C.c_int, C.c_float, vp]
            getattr(h, pre + "_lane_apply_preset_device").argtypes = [vp, u32, u32, u32, vp, C.c_size_t, vp, vp, C.c_float, vp]
            getattr(h, pre + "_lane_set_rate_device").argtypes = [vp, u32, u32, u32, vp, vp]
            getattr(h, pre + "_lane_collect_bulk_device").argtypes = [vp, u32, u32, u32, vp, vp, vp]
            getattr(h, pre + "_lane_collect_preset_device").argtypes = [vp, u32, u32, u32, vp, vp, C.c_size_t, vp]
            getattr(h, pre + "_lane_export_instances").argtypes = [vp, u32, u32, u32, vp, C.c_size_t]
            getattr(h, pre + "_lane_response_device").argtypes = [vp, u32, u32, u32, vp, u32, C.c_float, vp]
            getattr(h, pre + "_lane_get_preset_mute").argtypes = [vp, u32, u32, u32, vp]
            getattr(h, pre + "_lane_get_spdif_tx").argtypes = [vp, u32, u32, u32, vp]
            getattr(h, pre + "_lane_import_instances").argtypes = [vp, u32, u32, u32, vp, C.c_size_t]
            getattr(h, pre + "_lane_copy_instances").argtypes = [vp, u32, u32, u32, vp, vp]
        for pre in ("dspi_eq", "dspi_chain", "dspi_chainq"):
            getattr(h, pre + "_response_host").argtypes = [vp, u32, u32, vp, u32, C.c_float, vp]
            getattr(h, pre + "_response_device").argtypes = [vp, u32, u32, vp, u32, C.c_float, vp]
        h.dspi_eq_process_device_range.argtypes = [vp, vp, u32, u32, u32, u32]
        h.dspi_bind_host_to_device.argtypes = [C.c_int]
        h.dspi_nccl_unique_id.argtypes = [vp]
        h.dspi_sg_create.argtypes = [C.POINTER(vp), vp, C.c_int, vp, C.c_int, C.c_int, C.c_int]
        h.dspi_sg_destroy.argtypes = [vp]
        h.dspi_sg_process.argtypes = [vp, vp, u32, u32, u32]
        h.dspi_eqx_create.argtypes = [C.POINTER(vp), C.POINTER(_EqxDesc)]
        h.dspi_eqx_destroy.argtypes = [vp]
        h.dspi_eqx_shard_range.argtypes = [u32, u32, u32, vp, vp]
        h.dspi_eqx_upload_biquads.argtypes = [vp, u32, u32, vp]
        h.dspi_eqx_download_biquads.argtypes = [vp, u32, u32, vp]
        h.dspi_eqx_process_host.argtypes = [vp, vp, u32]
        h.dspi_eqx_process_root.argtypes = [vp, vp, u32, u32]
        h.dspi_eqx_launch_count.argtypes = [vp]
        h.dspi_eqx_launch_count.restype = C.c_uint64
        h.dspi_host_alloc.argtypes = [C.c_size_t]
        h.dspi_host_alloc.restype = vp
        h.dspi_host_free.argtypes = [vp]
        _lib = h
    return _lib


def _check(rc):
    if rc != 0:
        raise DspiError(f"dspi error {rc}: {lib().dspi_last_error().decode()}")


def compute_coefficients(params, q28=False, fs=48000.0, biquads=None):
    """Host-side ``dsp_compute_coefficients`` over an array of recipes.

    ``params``: EQ_PARAM array (clamped in place like the reference);
    ``biquads``: matching BIQUAD_* array to update (state kept) or None for fresh zeros.
    """
    h = lib()
    dt = L.BIQUAD_Q28 if q28 else L.BIQUAD_F32
    if biquads is None:
        biquads = np.zeros(params.shape, dt)
    fn = h.dspi_compute_coefficients_q28 if q28 else h.dspi_compute_coefficients_f32
    pp, bb = params.reshape(-1), biquads.reshape(-1)
    bp, bbp = pp.ctypes.data, bb.ctypes.data
    for i in range(pp.shape[0]):
        fn(bp + i * pp.dtype.itemsize, bbp + i * bb.dtype.itemsize, fs)
    return biquads


class PinnedBuffer:
    """Page-locked host memory viewed as a numpy array."""

    def __init__(self, shape, dtype):
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        self.ptr = lib().dspi_host_alloc(self.nbytes)
        if not self.ptr:
            raise DspiError("dspi_host_alloc failed")
        buf = (C.c_uint8 * self.nbytes).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype).reshape(self.shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().dspi_host_free(self.ptr)
            self.ptr = None


def _pinned(buf):
    """(address, bytes, rows) of a PinnedBuffer or a torch tensor (its memory is checked by the library, not here)"""
    if isinstance(buf, PinnedBuffer):
        return buf.ptr, buf.nbytes, buf.shape[0]
    if hasattr(buf, "data_ptr") and hasattr(buf, "is_contiguous"):
        if not buf.is_contiguous():
            raise ValueError("a host buffer must be contiguous")
        return buf.data_ptr(), buf.numel() * buf.element_size(), buf.shape[0]
    raise TypeError("a host buffer must be a PinnedBuffer or a pinned torch tensor")


class EqEngine:
    """Many independent 10-band cascades on one GPU (``dspi_eq_*``)."""

    def __init__(self, arith, n_channels, n_bands=L.NUM_BANDS, device=0):
        self.arith = ARITH[arith] if isinstance(arith, str) else int(arith)
        self.q28 = self.arith == ARITH_Q28
        self.n_channels, self.n_bands, self.device = int(n_channels), int(n_bands), int(device)
        self.biquad_dtype = L.BIQUAD_Q28 if self.q28 else L.BIQUAD_F32
        self.sample_dtype = np.int32 if self.q28 else np.float32
        self._h = C.c_void_p()
        desc = _EqDesc(self.arith, self.n_channels, self.n_bands, self.device, 0)
        _check(lib().dspi_eq_create(C.byref(self._h), C.byref(desc)))

    def close(self):
        if self._h:
            lib().dspi_eq_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, biquads, ch0=0):
        b = np.ascontiguousarray(biquads)
        assert b.dtype == self.biquad_dtype and b.ndim == 2 and b.shape[1] == L.MAX_BANDS
        _check(lib().dspi_eq_upload_biquads(self._h, ch0, b.shape[0], b.ctypes.data))

    def download(self, n=None, ch0=0):
        n = self.n_channels - ch0 if n is None else n
        out = np.zeros((n, L.MAX_BANDS), self.biquad_dtype)
        _check(lib().dspi_eq_download_biquads(self._h, ch0, n, out.ctypes.data))
        return out

    def set_param(self, channel, param, fs):
        p = np.array([param], dtype=L.EQ_PARAM) if not isinstance(param, np.ndarray) else param.reshape(1).copy()
        _check(lib().dspi_eq_set_param(self._h, channel, p.ctypes.data, fs))
        return p[0]

    def process_device(self, dev_ptr, T, ld=None):
        _check(lib().dspi_eq_process_device(self._h, C.c_void_p(int(dev_ptr)), T, T if ld is None else ld))

    def process_device_range(self, dev_ptr, T, ld, ch0, n):
        """Channels [ch0, ch0+n) only; ``dev_ptr`` is the row of channel ch0."""
        _check(lib().dspi_eq_process_device_range(self._h, C.c_void_p(int(dev_ptr)), int(T), int(ld), int(ch0), int(n)))

    def process_host(self, samples):
        """``samples``: C-contiguous [n_channels, T] numpy array (or PinnedBuffer.array); in place."""
        assert samples.flags["C_CONTIGUOUS"] and samples.dtype == self.sample_dtype and samples.shape[0] == self.n_channels
        _check(lib().dspi_eq_process_host(self._h, samples.ctypes.data, samples.shape[1]))

    def sync(self):
        _check(lib().dspi_eq_sync(self._h))

    @property
    def stream(self):
        return lib().dspi_eq_stream(self._h)

    @property
    def launch_count(self):
        return int(lib().dspi_eq_launch_count(self._h))

    def set_params_device(self, recipes, fs, ch0=0):
        """``dsp_compute_coefficients`` for every band of ``recipes`` (EQ_PARAM [n, 12]) on the GPU; returns the clamped recipes."""
        r = np.ascontiguousarray(recipes, L.EQ_PARAM).copy()
        assert r.ndim == 2 and r.shape[1] == L.MAX_BANDS
        _check(lib().dspi_eq_set_params_device(self._h, int(ch0), int(r.shape[0]), r.ctypes.data_as(C.c_void_p), C.c_float(fs)))
        return r

    def response(self, freqs, fs, ch0=0, n=None, out_ptr=0):
        """Frequency response of channels [ch0, ch0+n) at ``freqs`` (Hz): complex64 [n, n_freqs] (``dspi_eq_response_host``).
        With ``out_ptr`` (device memory for [n, n_freqs] complex64) it runs ``dspi_eq_response_device`` and returns None."""
        return _response(self._h, "dspi_eq", (), self.n_channels, freqs, fs, ch0, n, out_ptr)

    def kernel_info(self):
        """Which kernel the next process call runs (triggers a pending run-time specialisation)."""
        buf = C.create_string_buffer(320)
        _check(lib().dspi_eq_kernel_info(self._h, buf, len(buf)))
        return buf.value.decode()


class EqGroup:
    """The EQ engine over several GPUs of one box, one process (``dspi_eqx_*``): contiguous channel shards, no exchange."""

    def __init__(self, arith, n_channels, devices, n_bands=L.NUM_BANDS):
        self.arith = ARITH[arith] if isinstance(arith, str) else int(arith)
        self.q28 = self.arith == ARITH["q28"]
        self.n_channels, self.devices = int(n_channels), list(devices)
        d = _EqxDesc(self.arith, self.n_channels, int(n_bands), len(self.devices), (C.c_int32 * 8)(*(self.devices + [0] * (8 - len(self.devices)))), 0)
        self._h = C.c_void_p()
        _check(lib().dspi_eqx_create(C.byref(self._h), C.byref(d)))

    def close(self):
        if self._h:
            lib().dspi_eqx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def shard_range(self, k):
        lo, hi = C.c_uint32(), C.c_uint32()
        _check(lib().dspi_eqx_shard_range(self.n_channels, len(self.devices), k, C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    def upload(self, biquads, ch0=0):
        b = np.ascontiguousarray(biquads)
        _check(lib().dspi_eqx_upload_biquads(self._h, int(ch0), int(b.shape[0]), b.ctypes.data))

    def download(self, n=None, ch0=0):
        n = self.n_channels - ch0 if n is None else n
        out = np.zeros((n, L.MAX_BANDS), L.BIQUAD_Q28 if self.q28 else L.BIQUAD_F32)
        _check(lib().dspi_eqx_download_biquads(self._h, int(ch0), int(n), out.ctypes.data))
        return out

    def process_host(self, samples):
        assert samples.flags["C_CONTIGUOUS"] and samples.shape[0] == self.n_channels and samples.dtype.itemsize == 4
        _check(lib().dspi_eqx_process_host(self._h, samples.ctypes.data, int(samples.shape[1])))

    def process_root(self, dev_ptr, T, ld=None):
        _check(lib().dspi_eqx_process_root(self._h, C.c_void_p(int(dev_ptr)), int(T), int(T if ld is None else ld)))

    @property
    def launch_count(self):
        return int(lib().dspi_eqx_launch_count(self._h))


def nccl_unique_id():
    """128-byte NCCL unique id (call on one rank, hand the bytes to the others)."""
    buf = (C.c_uint8 * 128)()
    _check(lib().dspi_nccl_unique_id(buf))
    return bytes(buf)


class ScatterGather:
    """One rank's end of the native NCCL scatter / process / gather pipeline (``dspi_sg_*``) around an :class:`EqEngine`."""

    def __init__(self, engine, device, unique_id, rank, world, root=0):
        self._h = C.c_void_p()
        self.engine = engine
        idb = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        _check(lib().dspi_sg_create(C.byref(self._h), engine._h, int(device), idb, int(rank), int(world), int(root)))

    def process(self, full_ptr, total_channels, T, n_chunks=0):
        _check(lib().dspi_sg_process(self._h, C.c_void_p(int(full_ptr)) if full_ptr else None, int(total_channels), int(T), int(n_chunks)))

    def close(self):
        if self._h:
            lib().dspi_sg_destroy(self._h)
            self._h = C.c_void_p()


def _packet_table(packet_frames):
    """Any integer sequence of packet lengths -> (uint16 array, total frames).  The library rejects lengths outside
    1..192; values that would wrap in uint16 are rejected here."""
    t = np.asarray(packet_frames, np.int64).reshape(-1)
    if t.size and (t.min() < 0 or t.max() > 0xFFFF):
        raise DspiError("packet lengths must be 1..192 frames")
    t = np.ascontiguousarray(t, np.uint16)
    return t, int(t.sum(dtype=np.int64))


def _response(h, pre, shape, n_total, freqs, fs, first, n, out_ptr):
    """Shared body of the ``response`` methods: complex64 [n, *shape, n_freqs] from ``*_response_host``, or None after
    ``*_response_device`` into ``out_ptr`` (device memory, asynchronous on the engine stream)."""
    f = np.ascontiguousarray(freqs, np.float32).reshape(-1)
    n = n_total - first if n is None else int(n)
    if out_ptr:
        _check(getattr(lib(), pre + "_response_device")(h, int(first), n, f.ctypes.data, f.size, C.c_float(fs), C.c_void_p(int(out_ptr))))
        return None
    out = np.zeros((max(n, 0),) + tuple(shape) + (f.size,), np.complex64)
    _check(getattr(lib(), pre + "_response_host")(h, int(first), n, f.ctypes.data, f.size, C.c_float(fs), out.ctypes.data))
    return out


def bind_host_to_device(device):
    """NUMA-bind this thread and its future allocations to the device's PCIe node; returns the node or -1."""
    return int(lib().dspi_bind_host_to_device(int(device)))


class _ChainEngine:
    """What both chain engines share; the subclasses differ in their constructor and in their class attributes (the
    C prefix ``_PRE``, the ``_PARAMS``, ``_BIQUAD`` and ``_STATUS`` dtypes, EQ channels ``_ROLES``, outputs ``_OUTS``, S/PDIF
    pairs ``_PAIRS`` and the preset slot ``_PLATFORM``)."""

    def _fn(self, name):
        return getattr(lib(), self._PRE + "_" + name)

    def close(self):
        if self._h:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_params(self, params, inst0=0):
        p = np.ascontiguousarray(params)
        assert p.dtype == self._PARAMS and p.ndim == 1
        _check(self._fn("set_params")(self._h, inst0, p.shape[0], p.ctypes.data))

    def upload_biquads(self, biquads, inst0=0):
        b = np.ascontiguousarray(biquads)
        assert b.dtype == self._BIQUAD and b.shape[1:] == (self._ROLES, L.MAX_BANDS)
        _check(self._fn("upload_biquads")(self._h, inst0, b.shape[0], b.ctypes.data))

    def set_eq_params_device(self, recipes, fs, inst0=0):
        """EQ_PARAM [n, roles, 12] -> coefficients of all bands computed on the GPU; returns the clamped recipes."""
        r = np.ascontiguousarray(recipes, L.EQ_PARAM).copy()
        assert r.shape[1:] == (self._ROLES, L.MAX_BANDS)
        _check(self._fn("set_eq_params_device")(self._h, int(inst0), int(r.shape[0]), r.ctypes.data_as(C.c_void_p), C.c_float(fs)))
        return r

    def download_biquads(self, n=None, inst0=0):
        n = self.n_instances - inst0 if n is None else n
        out = np.zeros((n, self._ROLES, L.MAX_BANDS), self._BIQUAD)
        _check(self._fn("download_biquads")(self._h, inst0, n, out.ctypes.data))
        return out

    def state_export(self):
        """Checkpoint: filter / leveller / delay / modulator state (and coefficients) as one bytes-like blob."""
        n = int(self._fn("state_size")(self._h))
        blob = np.zeros(n, np.uint8)
        _check(self._fn("state_export")(self._h, blob.ctypes.data_as(C.c_void_p), C.c_size_t(n)))
        return blob

    def state_import(self, blob):
        b = np.ascontiguousarray(blob, np.uint8)
        _check(self._fn("state_import")(self._h, b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size)))

    def instance_image_size(self):
        """Bytes of one instance image (``export_instances``)."""
        return int(self._fn("instance_image_size")(self._h))

    def export_instances(self, inst0=0, n=None):
        """Images of instances [inst0, inst0+n) (default: to the end), uint8 [n, instance_image_size]: everything of each
        instance a later call depends on - parameters, biquads and all running state, S/PDIF transmitter, configuration
        record.  Ordered behind earlier work on the engine stream; changes nothing."""
        n = self.n_instances - int(inst0) if n is None else int(n)
        size = self.instance_image_size()
        out = np.zeros((max(n, 0), size), np.uint8)
        _check(self._fn("export_instances")(self._h, int(inst0), n, out.ctypes.data_as(C.c_void_p), C.c_size_t(size)))
        return out

    def import_instances(self, images, inst0=0):
        """uint8 [n, stride] images (stride >= instance_image_size) from an engine of the same arith and band count, any
        size or device -> instances [inst0, inst0+n), from the next process call on.  All or nothing: a bad header raises
        and writes nothing."""
        img = np.ascontiguousarray(images, np.uint8)
        if img.ndim != 2:
            raise ValueError("images must be [n, stride] bytes")
        _check(self._fn("import_instances")(self._h, int(inst0), int(img.shape[0]), img.ctypes.data_as(C.c_void_p),
                                            C.c_size_t(img.shape[1])))

    def copy_instances(self, src, dst):
        """Instance ``src[k]`` -> instance ``dst[k]`` on the GPU, as ``export_instances(src[k], 1)`` then
        ``import_instances(..., dst[k])`` would, with no image leaving the device.  ``src`` may repeat; ``dst`` must be
        distinct and share no index with ``src``.  Ordered behind earlier work; returns when the engine is updated."""
        s, d = self._copy_lists(src, dst)
        _check(self._fn("copy_instances")(self._h, int(s.size), s.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p)))

    @staticmethod
    def _copy_lists(src, dst):
        s = np.ascontiguousarray(np.asarray(src, np.int64).reshape(-1))
        d = np.ascontiguousarray(np.asarray(dst, np.int64).reshape(-1))
        if s.shape != d.shape:
            raise ValueError("src and dst give different copy counts")
        if s.size and (min(s.min(), d.min()) < 0 or max(s.max(), d.max()) > 0xFFFFFFFF):
            raise ValueError("instance indices must be 0 .. 2**32 - 1")
        return s.astype(np.uint32), d.astype(np.uint32)

    def reset_instances(self, inst0=0, n=None):
        """``reset_state`` for instances [inst0, inst0+n) only (default: to the end); parameters are kept."""
        n = self.n_instances - int(inst0) if n is None else int(n)
        _check(self._fn("reset_instances")(self._h, int(inst0), n))

    def sm_partition(self):
        """(SMs reserved for the modulator, SMs for every other stage); (0, 0) without a partition."""
        a, b = C.c_uint32(), C.c_uint32()
        _check(self._fn("sm_partition")(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def set_dynamics_device(self, cfgs, fs, inst0=0):
        """DYNAMICS_CONFIG [n]: crossfeed / leveller / loudness coefficients and the host volume generated on the GPU."""
        cf = np.ascontiguousarray(cfgs, L.DYNAMICS_CONFIG)
        _check(self._fn("set_dynamics_device")(self._h, int(inst0), int(cf.shape[0]), cf.ctypes.data_as(C.c_void_p), C.c_float(fs)))

    def set_preset_mute(self, states, fs, inst0=0, n=None):
        """Envelope mode for instances [inst0, inst0+n): ``states`` PRESET_MUTE [n], or None to leave envelope mode."""
        if states is None:
            n = self.n_instances - inst0 if n is None else n
            _check(self._fn("set_preset_mute")(self._h, int(inst0), int(n), None, int(fs)))
            return
        st = np.ascontiguousarray(states, L.PRESET_MUTE)
        _check(self._fn("set_preset_mute")(self._h, int(inst0), int(st.shape[0]), st.ctypes.data_as(C.c_void_p), int(fs)))

    def get_preset_mute(self, n=None, inst0=0):
        n = self.n_instances - inst0 if n is None else n
        out = np.zeros(n, L.PRESET_MUTE)
        _check(self._fn("get_preset_mute")(self._h, int(inst0), int(n), out.ctypes.data_as(C.c_void_p)))
        return out

    def reset_state(self):
        _check(self._fn("reset_state")(self._h))

    def process_host(self, pcm, bit_depth, n_packets, frames_per_packet, want_spdif=True, want_pdm=True, want_status=True):
        """``pcm``: uint8 [n_instances, n_frames * bytes_per_frame].  Returns (spdif, pdm, status)."""
        return self._process_host("process_host", pcm, bit_depth, n_packets * frames_per_packet, (n_packets, frames_per_packet),
                                  want_spdif, want_pdm, want_status)

    def process_device(self, pcm_ptr, bit_depth, n_packets, frames_per_packet, spdif_ptr=0, pdm_ptr=0, status_ptr=0):
        _check(self._fn("process_device")(self._h, C.c_void_p(int(pcm_ptr)), bit_depth, n_packets, frames_per_packet,
                                          C.c_void_p(int(spdif_ptr)) if spdif_ptr else None,
                                          C.c_void_p(int(pdm_ptr)) if pdm_ptr else None,
                                          C.c_void_p(int(status_ptr)) if status_ptr else None))

    def process_packets_host(self, pcm, bit_depth, packet_frames, want_spdif=True, want_pdm=True, want_status=True):
        """One USB packet per entry of ``packet_frames`` (its length in frames, shared by every instance).
        ``pcm``: uint8 [n_instances, F * bytes_per_frame] with F = sum(packet_frames).  Returns (spdif, pdm, status), spdif
        int32 [n_instances, S/PDIF pairs, F, 2]."""
        t, F = _packet_table(packet_frames)
        return self._process_host("process_packets_host", pcm, bit_depth, F, (t.size, t.ctypes.data), want_spdif, want_pdm, want_status)

    def process_packets_range_host(self, inst0, pcm, bit_depth, packet_frames, want_spdif=True, want_pdm=True, want_status=True):
        """``process_packets_host`` over instances [inst0, inst0 + n) only, n = ``pcm.shape[0]`` (inst0 a multiple of 64),
        with this call's own ``packet_frames``.  Every array has n rows, row i for instance inst0 + i; nothing outside the
        range changes.  Returns (spdif, pdm, status)."""
        t, F = _packet_table(packet_frames)
        pcm = np.ascontiguousarray(pcm)
        n = pcm.shape[0]
        assert pcm.dtype == np.uint8 and pcm.shape == (n, F * (6 if bit_depth == 24 else 4))
        spdif = np.zeros((n, self._PAIRS, F, 2), np.int32) if want_spdif else None
        pdm = np.zeros((n, F, 8), np.uint32) if want_pdm else None
        status = np.zeros(n, self._STATUS) if want_status else None
        _check(self._fn("process_packets_range_host")(self._h, int(inst0), n, pcm.ctypes.data, bit_depth, t.size, t.ctypes.data,
                                                      spdif.ctypes.data if want_spdif else None, pdm.ctypes.data if want_pdm else None,
                                                      status.ctypes.data if want_status else None))
        return spdif, pdm, status

    def process_packets_range_device(self, inst0, n, pcm_ptr, bit_depth, packet_frames, spdif_ptr=0, pdm_ptr=0, status_ptr=0):
        """``process_packets_range_host`` with device pointers to n-row buffers, asynchronous on the engine stream."""
        t, _ = _packet_table(packet_frames)
        _check(self._fn("process_packets_range_device")(self._h, int(inst0), int(n), C.c_void_p(int(pcm_ptr)), bit_depth, t.size, t.ctypes.data,
                                                        C.c_void_p(int(spdif_ptr)) if spdif_ptr else None,
                                                        C.c_void_p(int(pdm_ptr)) if pdm_ptr else None,
                                                        C.c_void_p(int(status_ptr)) if status_ptr else None))

    def _process_host(self, name, pcm, bit_depth, F, schedule, want_spdif, want_pdm, want_status):
        pcm = np.ascontiguousarray(pcm)
        assert pcm.dtype == np.uint8 and pcm.shape == (self.n_instances, F * (6 if bit_depth == 24 else 4))
        spdif = np.zeros((self.n_instances, self._PAIRS, F, 2), np.int32) if want_spdif else None
        pdm = np.zeros((self.n_instances, F, 8), np.uint32) if want_pdm else None
        status = np.zeros(self.n_instances, self._STATUS) if want_status else None
        _check(self._fn(name)(self._h, pcm.ctypes.data, bit_depth, *schedule,
                              spdif.ctypes.data if want_spdif else None, pdm.ctypes.data if want_pdm else None,
                              status.ctypes.data if want_status else None))
        return spdif, pdm, status

    def process_packets_device(self, pcm_ptr, bit_depth, packet_frames, spdif_ptr=0, pdm_ptr=0, status_ptr=0):
        """``process_packets_host`` with device pointers, asynchronous on the engine stream (outputs for F = sum(packet_frames))."""
        t, _ = _packet_table(packet_frames)
        _check(self._fn("process_packets_device")(self._h, C.c_void_p(int(pcm_ptr)), bit_depth, t.size, t.ctypes.data,
                                                  C.c_void_p(int(spdif_ptr)) if spdif_ptr else None,
                                                  C.c_void_p(int(pdm_ptr)) if pdm_ptr else None,
                                                  C.c_void_p(int(status_ptr)) if status_ptr else None))

    def response(self, freqs, fs, inst0=0, n=None, out_ptr=0):
        """Frequency response of instances [inst0, inst0+n): complex64 [n, outputs, 2 inputs, n_freqs]; with ``out_ptr``
        (device memory) asynchronous on the engine stream, returning None."""
        return _response(self._h, self._PRE, (self._OUTS, 2), self.n_instances, freqs, fs, inst0, n, out_ptr)

    def sync(self):
        _check(self._fn("sync")(self._h))

    @property
    def stream(self):
        return self._fn("stream")(self._h)

    @property
    def launch_count(self):
        return int(self._fn("launch_count")(self._h))

    def apply_bulk_device(self, packets, fs, inst0=0, host=None, exact_db=False):
        """WIRE_BULK [n] -> instances [inst0, inst0+n) reconfigured on the GPU as ``bulk_params_apply`` and the firmware's main
        loop would; ``host`` BULK_HOST [n] (default: volume 0 dB, not muted).  Returns the firmware's result codes, int32 [n]:
        0 applied, -1 .. -4 rejected (that instance is left exactly as it was)."""
        w, hv = self._bulk_args(packets, host)
        res = np.zeros(w.shape[0], np.int32)
        _check(self._fn("apply_bulk_device")(self._h, int(inst0), int(w.shape[0]), w.ctypes.data_as(C.c_void_p),
                                             hv.ctypes.data_as(C.c_void_p), int(bool(exact_db)), C.c_float(fs),
                                             res.ctypes.data_as(C.c_void_p)))
        return res

    @staticmethod
    def _bulk_args(packets, host):
        w = np.ascontiguousarray(packets, L.WIRE_BULK).reshape(-1)
        hv = np.zeros(w.shape[0], L.BULK_HOST) if host is None else np.ascontiguousarray(host, L.BULK_HOST).reshape(-1)
        if hv.shape[0] != w.shape[0]:
            raise ValueError("packets and host give different instance counts")
        return w, hv

    def set_rate_device(self, rates, inst0=0):
        """The USB host switched instances [inst0, inst0+n) to ``rates`` (float [n], one rate per instance, or a scalar for
        one instance): every rate-dependent record re-derived on the GPU from each instance's configuration record, as
        ``perform_rate_change`` does.  Returns int32 [n] of ``layouts.BULK_*`` marks; only ``BULK_CURRENT`` instances switched,
        the others are left exactly as they were."""
        r = np.ascontiguousarray(np.asarray(rates, np.float32).reshape(-1))
        res = np.zeros(r.size, np.int32)
        _check(self._fn("set_rate_device")(self._h, int(inst0), int(r.size), r.ctypes.data_as(C.c_void_p), res.ctypes.data_as(C.c_void_p)))
        return res

    def edit_bulk_device(self, edits, fs, exact_db=False):
        """BULK_EDIT [n] (see ``layouts.bulk_edit``) -> single fields of current instances edited on the GPU, in list order,
        as collect + patch + ``apply_bulk_device(fs, exact_db)`` would leave them, with only the touched fields re-derived.
        Returns int32 [n]: the ``layouts.BULK_*`` mark of each edit's instance; stale and unset instances are left alone."""
        e = np.ascontiguousarray(edits, L.BULK_EDIT).reshape(-1)
        res = np.zeros(e.shape[0], np.int32)
        _check(self._fn("edit_bulk_device")(self._h, int(e.shape[0]), e.ctypes.data_as(C.c_void_p), int(bool(exact_db)), C.c_float(fs),
                                            res.ctypes.data_as(C.c_void_p)))
        return res

    def collect_bulk_device(self, inst0=0, n=None):
        """``REQ_GET_ALL_PARAMS`` for instances [inst0, inst0+n) (default: to the end) from the engine's configuration records:
        (WIRE_BULK [n], BULK_HOST [n], int32 [n] of ``layouts.BULK_CURRENT`` / ``BULK_STALE`` / ``BULK_UNSET``).  A current or
        stale packet is what ``bulk_params_collect`` returns for the host state the same calls would have left; an unset
        instance gives zero bytes."""
        n = self.n_instances - int(inst0) if n is None else int(n)
        w, hv, res = np.zeros(max(n, 0), L.WIRE_BULK), np.zeros(max(n, 0), L.BULK_HOST), np.zeros(max(n, 0), np.int32)
        _check(self._fn("collect_bulk_device")(self._h, int(inst0), n, w.ctypes.data_as(C.c_void_p),
                                               hv.ctypes.data_as(C.c_void_p), res.ctypes.data_as(C.c_void_p)))
        return w, hv, res

    def apply_preset_device(self, images, fs, inst0=0, slots=0, master_volume_mode=0, dir_master_volume_db=0.0, host=None):
        """uint8 [n, stride] slot images (stride >= ``preset_slot_size``, e.g. 4096-byte flash sectors) -> instances
        [inst0, inst0+n) reconfigured on the GPU as ``preset_load`` and the firmware's main loop would.  ``slots``,
        ``master_volume_mode`` and ``dir_master_volume_db`` are scalars or [n]; ``host`` BULK_HOST [n] (default: volume 0 dB,
        not muted).  Returns int32 [n]: 0 loaded, 3 (PRESET_ERR_CRC) rejected (that instance is left exactly as it was)."""
        img, ld, hv = self._preset_args(images, slots, master_volume_mode, dir_master_volume_db, host)
        n = img.shape[0]
        res = np.zeros(n, np.int32)
        _check(self._fn("apply_preset_device")(self._h, int(inst0), n, img.ctypes.data_as(C.c_void_p), C.c_size_t(img.shape[1]),
                                               ld.ctypes.data_as(C.c_void_p), hv.ctypes.data_as(C.c_void_p), C.c_float(fs),
                                               res.ctypes.data_as(C.c_void_p)))
        return res

    @staticmethod
    def _preset_args(images, slots, master_volume_mode, dir_master_volume_db, host):
        img = np.ascontiguousarray(images, np.uint8)
        if img.ndim != 2:
            raise ValueError("images must be [n, stride] bytes")
        n = img.shape[0]
        ld = np.zeros(n, L.PRESET_LOAD)
        ld["slot_index"], ld["master_volume_mode"], ld["dir_master_volume_db"] = slots, master_volume_mode, dir_master_volume_db
        hv = np.zeros(n, L.BULK_HOST) if host is None else np.ascontiguousarray(host, L.BULK_HOST).reshape(-1)
        if hv.shape[0] != n:
            raise ValueError("images and host give different instance counts")
        return img, ld, hv

    def collect_preset_device(self, slots, inst0=0, n=None):
        """The state part of ``preset_save`` for instances [inst0, inst0+n) (default: as many as ``slots`` gives, or to the
        end for a scalar): (uint8 [n, slot size] images, int32 [n] of ``layouts.BULK_*`` marks).  An unset instance gives zero
        bytes."""
        sl = np.asarray(slots, np.uint8).reshape(-1)
        n = (self.n_instances - int(inst0) if sl.size == 1 else sl.size) if n is None else int(n)
        sl = np.ascontiguousarray(np.broadcast_to(sl, (max(n, 0),)) if sl.size == 1 else sl)
        if sl.size != max(n, 0):
            raise ValueError("slots and n give different instance counts")
        size = preset_slot_size(self._PLATFORM)
        img, res = np.zeros((max(n, 0), size), np.uint8), np.zeros(max(n, 0), np.int32)
        _check(self._fn("collect_preset_device")(self._h, int(inst0), n, sl.ctypes.data_as(C.c_void_p), img.ctypes.data_as(C.c_void_p),
                                                 C.c_size_t(size), res.ctypes.data_as(C.c_void_p)))
        return img, res

    def set_spdif_tx(self, block_pos, channel_status, inst0=0):
        """Transmitter state of instances [inst0, inst0+n): ``block_pos`` an int or [n] (0..191), ``channel_status`` 5 bytes
        or uint8 [n, 5]; a single value on either side applies to all n.  Takes effect from the next process call."""
        rec = self._spdif_records(block_pos, channel_status)
        _check(self._fn("set_spdif_tx")(self._h, int(inst0), int(rec.size), rec.ctypes.data_as(C.c_void_p)))

    @staticmethod
    def _spdif_records(block_pos, channel_status):
        bp = np.asarray(block_pos, np.int64).reshape(-1)
        cs = np.frombuffer(bytes(channel_status), np.uint8) if isinstance(channel_status, (bytes, bytearray)) else np.asarray(channel_status, np.uint8)
        cs = cs.reshape(-1, 5)
        n = max(bp.size, cs.shape[0])
        if bp.size not in (1, n) or cs.shape[0] not in (1, n):
            raise ValueError("block_pos and channel_status give different instance counts")
        if bp.size and (bp.min() < 0 or bp.max() > 255):
            raise DspiError("block_pos must be 0..191")
        rec = np.zeros(n, L.SPDIF_TX)
        rec["block_pos"] = bp
        rec["channel_status"] = cs
        return rec

    def get_spdif_tx(self, n=None, inst0=0):
        """SPDIF_TX [n]: block position of the next frame and channel status, after the last call issued."""
        n = self.n_instances - inst0 if n is None else n
        out = np.zeros(n, L.SPDIF_TX)
        _check(self._fn("get_spdif_tx")(self._h, int(inst0), int(n), out.ctypes.data_as(C.c_void_p)))
        return out

    def process_subframes_host(self, pcm, bit_depth, packet_frames, want_subframes=True, want_pdm=True, want_status=True):
        """As ``process_packets_host``, S/PDIF out as subframes: uint32 [n_instances, pairs, F, 2, 2] ({l, h} per subframe,
        the array ``spdif_encode_host`` makes of the words, reshaped).  Returns (subframes, pdm, status)."""
        t, F = _packet_table(packet_frames)
        pcm = np.ascontiguousarray(pcm)
        assert pcm.dtype == np.uint8 and pcm.shape == (self.n_instances, F * (6 if bit_depth == 24 else 4))
        sub = np.zeros((self.n_instances, self._PAIRS, F, 2, 2), np.uint32) if want_subframes else None
        pdm = np.zeros((self.n_instances, F, 8), np.uint32) if want_pdm else None
        status = np.zeros(self.n_instances, self._STATUS) if want_status else None
        _check(self._fn("process_subframes_host")(self._h, pcm.ctypes.data, bit_depth, t.size, t.ctypes.data,
                                                  sub.ctypes.data if want_subframes else None,
                                                  pdm.ctypes.data if want_pdm else None,
                                                  status.ctypes.data if want_status else None))
        return sub, pdm, status

    def process_subframes_range_host(self, inst0, pcm, bit_depth, packet_frames, want_subframes=True, want_pdm=True, want_status=True):
        """``process_subframes_host`` over instances [inst0, inst0 + n) only, n = ``pcm.shape[0]``, as
        ``process_packets_range_host``.  Returns (subframes, pdm, status) with n rows each."""
        t, F = _packet_table(packet_frames)
        pcm = np.ascontiguousarray(pcm)
        n = pcm.shape[0]
        assert pcm.dtype == np.uint8 and pcm.shape == (n, F * (6 if bit_depth == 24 else 4))
        sub = np.zeros((n, self._PAIRS, F, 2, 2), np.uint32) if want_subframes else None
        pdm = np.zeros((n, F, 8), np.uint32) if want_pdm else None
        status = np.zeros(n, self._STATUS) if want_status else None
        _check(self._fn("process_subframes_range_host")(self._h, int(inst0), n, pcm.ctypes.data, bit_depth, t.size, t.ctypes.data,
                                                        sub.ctypes.data if want_subframes else None,
                                                        pdm.ctypes.data if want_pdm else None,
                                                        status.ctypes.data if want_status else None))
        return sub, pdm, status

    def process_subframes_range_device(self, inst0, n, pcm_ptr, bit_depth, packet_frames, subframes_ptr=0, pdm_ptr=0, status_ptr=0):
        """``process_subframes_range_host`` with device pointers (subframes 16-byte aligned), asynchronous on the engine stream."""
        t, _ = _packet_table(packet_frames)
        _check(self._fn("process_subframes_range_device")(self._h, int(inst0), int(n), C.c_void_p(int(pcm_ptr)), bit_depth, t.size, t.ctypes.data,
                                                          C.c_void_p(int(subframes_ptr)) if subframes_ptr else None,
                                                          C.c_void_p(int(pdm_ptr)) if pdm_ptr else None,
                                                          C.c_void_p(int(status_ptr)) if status_ptr else None))

    def process_subframes_device(self, pcm_ptr, bit_depth, packet_frames, subframes_ptr=0, pdm_ptr=0, status_ptr=0):
        """``process_subframes_host`` with device pointers (subframes 16-byte aligned), asynchronous on the engine stream."""
        t, _ = _packet_table(packet_frames)
        _check(self._fn("process_subframes_device")(self._h, C.c_void_p(int(pcm_ptr)), bit_depth, t.size, t.ctypes.data,
                                                    C.c_void_p(int(subframes_ptr)) if subframes_ptr else None,
                                                    C.c_void_p(int(pdm_ptr)) if pdm_ptr else None,
                                                    C.c_void_p(int(status_ptr)) if status_ptr else None))

    def lane_open(self, inst0, n):
        """Open a lane over instances [inst0, inst0+n) (inst0 a multiple of 64, no overlap with an open lane's window): an issue
        queue whose calls run concurrently with other lanes' calls.  Returns the lane id."""
        lane = C.c_uint32()
        _check(self._fn("lane_open")(self._h, int(inst0), int(n), C.byref(lane)))
        return lane.value

    def lane_close(self, lane):
        """Wait for the lane's calls and free its streams."""
        _check(self._fn("lane_close")(self._h, int(lane)))

    def _lane_process(self, form, lane, inst0, n, pcm_ptr, bit_depth, packet_frames, out_ptr, pdm_ptr, status_ptr):
        t, _ = _packet_table(packet_frames)
        _check(self._fn("lane_process_%s_device" % form)(self._h, int(lane), int(inst0), int(n), C.c_void_p(int(pcm_ptr)), bit_depth, t.size,
                                                         t.ctypes.data, C.c_void_p(int(out_ptr)) if out_ptr else None,
                                                         C.c_void_p(int(pdm_ptr)) if pdm_ptr else None,
                                                         C.c_void_p(int(status_ptr)) if status_ptr else None))

    def lane_process_packets_device(self, lane, inst0, n, pcm_ptr, bit_depth, packet_frames, spdif_ptr=0, pdm_ptr=0, status_ptr=0):
        """``process_packets_range_device`` issued on a lane (the range inside its window), asynchronous on ``lane_stream(lane)``."""
        self._lane_process("packets", lane, inst0, n, pcm_ptr, bit_depth, packet_frames, spdif_ptr, pdm_ptr, status_ptr)

    def lane_process_subframes_device(self, lane, inst0, n, pcm_ptr, bit_depth, packet_frames, subframes_ptr=0, pdm_ptr=0, status_ptr=0):
        """``process_subframes_range_device`` issued on a lane (the range inside its window), asynchronous on ``lane_stream(lane)``."""
        self._lane_process("subframes", lane, inst0, n, pcm_ptr, bit_depth, packet_frames, subframes_ptr, pdm_ptr, status_ptr)

    def lane_process_packets_host(self, lane, inst0, pcm, bit_depth, packet_frames, spdif=None, pdm=None, status=None, subframes=False):
        """``process_packets_range_host`` (``subframes``: ``process_subframes_range_host``) issued on a lane, over
        [inst0, inst0 + n) inside its window, n = rows of ``pcm``.  Every buffer is page-locked host memory: a ``PinnedBuffer``
        or a pinned torch tensor (pageable memory is refused).  ``pcm`` uint8 [n, F * bytes_per_frame]; ``spdif`` [n, pairs, F,
        2] int32 words or [n, pairs, F, 2, 2] uint32 subframes, ``pdm`` [n, F, 8] uint32 and ``status`` [n] status records,
        each optional.  Returns without waiting: ``pcm`` is read and the outputs are written on ``lane_stream(lane)``, so
        reuse ``pcm`` and read the outputs only after an event recorded there (or ``lane_sync``)."""
        t, F = _packet_table(packet_frames)
        p, nbytes, n = _pinned(pcm)
        if nbytes != n * F * (6 if bit_depth == 24 else 4):
            raise ValueError("pcm must hold n rows of F frames")
        need = [n * self._PAIRS * F * (16 if subframes else 8), n * F * 32, n * self._STATUS.itemsize]
        outs = []
        for buf, want, what in zip((spdif, pdm, status), need, ("spdif", "pdm", "status")):
            if buf is None:
                outs.append(None)
                continue
            ptr, size, _ = _pinned(buf)
            if size < want:
                raise ValueError("%s holds %d bytes, the call writes %d" % (what, size, want))
            outs.append(C.c_void_p(ptr))
        form = "subframes" if subframes else "packets"
        _check(self._fn("lane_process_%s_host" % form)(self._h, int(lane), int(inst0), n, C.c_void_p(p), bit_depth, t.size, t.ctypes.data, *outs))

    def lane_stream(self, lane):
        """The stream where the lane's outputs become visible (None for a lane that is not open)."""
        return self._fn("lane_stream")(self._h, int(lane))

    def lane_sync(self, lane):
        _check(self._fn("lane_sync")(self._h, int(lane)))

    def lane_edit_bulk_device(self, lane, edits, fs, exact_db=False, results_ptr=0):
        """``edit_bulk_device`` issued on a lane (every edit's instance inside its window), asynchronous on
        ``lane_stream(lane)``: returns without waiting.  ``results_ptr`` (device memory, int32 [n], or 0) receives the
        ``layouts.BULK_*`` mark of each edit's instance there."""
        e = np.ascontiguousarray(edits, L.BULK_EDIT).reshape(-1)
        _check(self._fn("lane_edit_bulk_device")(self._h, int(lane), int(e.shape[0]), e.ctypes.data_as(C.c_void_p), int(bool(exact_db)),
                                                 C.c_float(fs), C.c_void_p(int(results_ptr)) if results_ptr else None))

    def lane_set_preset_mute(self, lane, states, fs, inst0, n=None):
        """``set_preset_mute`` issued on a lane ([inst0, inst0+n) inside its window): ``states`` PRESET_MUTE [n] arms the
        fades, None (with ``n``) leaves envelope mode.  Asynchronous on ``lane_stream(lane)``."""
        if states is None:
            _check(self._fn("lane_set_preset_mute")(self._h, int(lane), int(inst0), int(n), None, int(fs)))
            return
        st = np.ascontiguousarray(states, L.PRESET_MUTE).reshape(-1)
        _check(self._fn("lane_set_preset_mute")(self._h, int(lane), int(inst0), int(st.shape[0]), st.ctypes.data_as(C.c_void_p), int(fs)))

    def lane_set_spdif_tx(self, lane, block_pos, channel_status, inst0):
        """``set_spdif_tx`` issued on a lane ([inst0, inst0+n) inside its window), asynchronous on ``lane_stream(lane)``."""
        rec = self._spdif_records(block_pos, channel_status)
        _check(self._fn("lane_set_spdif_tx")(self._h, int(lane), int(inst0), int(rec.size), rec.ctypes.data_as(C.c_void_p)))

    def lane_reset_instances(self, lane, inst0, n):
        """``reset_instances`` issued on a lane ([inst0, inst0+n) inside its window), asynchronous on ``lane_stream(lane)``."""
        _check(self._fn("lane_reset_instances")(self._h, int(lane), int(inst0), int(n)))

    def lane_apply_bulk_device(self, lane, packets, fs, inst0, host=None, exact_db=False, results_ptr=0):
        """``apply_bulk_device`` issued on a lane ([inst0, inst0+n) inside its window), asynchronous on ``lane_stream(lane)``:
        returns without waiting.  ``results_ptr`` (device memory, int32 [n], required) receives the firmware's result codes
        there."""
        w, hv = self._bulk_args(packets, host)
        _check(self._fn("lane_apply_bulk_device")(self._h, int(lane), int(inst0), int(w.shape[0]), w.ctypes.data_as(C.c_void_p),
                                                  hv.ctypes.data_as(C.c_void_p), int(bool(exact_db)), C.c_float(fs),
                                                  C.c_void_p(int(results_ptr)) if results_ptr else None))

    def lane_apply_preset_device(self, lane, images, fs, inst0, slots=0, master_volume_mode=0, dir_master_volume_db=0.0, host=None,
                                 results_ptr=0):
        """``apply_preset_device`` issued on a lane ([inst0, inst0+n) inside its window), asynchronous on ``lane_stream(lane)``:
        returns without waiting.  ``results_ptr`` (device memory, int32 [n], required) receives the preset result codes there."""
        img, ld, hv = self._preset_args(images, slots, master_volume_mode, dir_master_volume_db, host)
        _check(self._fn("lane_apply_preset_device")(self._h, int(lane), int(inst0), int(img.shape[0]), img.ctypes.data_as(C.c_void_p),
                                                    C.c_size_t(img.shape[1]), ld.ctypes.data_as(C.c_void_p), hv.ctypes.data_as(C.c_void_p),
                                                    C.c_float(fs), C.c_void_p(int(results_ptr)) if results_ptr else None))

    def lane_set_rate_device(self, lane, rates, inst0, results_ptr=0):
        """``set_rate_device`` issued on a lane ([inst0, inst0+n) inside its window), asynchronous on ``lane_stream(lane)``:
        returns without waiting.  ``results_ptr`` (device memory, int32 [n], or 0) receives the ``layouts.BULK_*`` marks there."""
        r = np.ascontiguousarray(np.asarray(rates, np.float32).reshape(-1))
        _check(self._fn("lane_set_rate_device")(self._h, int(lane), int(inst0), int(r.size), r.ctypes.data_as(C.c_void_p),
                                                C.c_void_p(int(results_ptr)) if results_ptr else None))

    # Lane reads: each writes what its engine-level counterpart returns into device memory on ``lane_stream(lane)`` and
    # returns without waiting; [inst0, inst0+n) lies inside the lane's window.

    def lane_collect_bulk_device(self, lane, inst0, n, packets_ptr, host_ptr=0, results_ptr=0):
        """``collect_bulk_device`` issued on a lane: WIRE_BULK [n] at ``packets_ptr``, BULK_HOST [n] at ``host_ptr`` and int32
        [n] marks at ``results_ptr`` (both optional)."""
        _check(self._fn("lane_collect_bulk_device")(self._h, int(lane), int(inst0), int(n), C.c_void_p(int(packets_ptr)) if packets_ptr else None,
                                                    C.c_void_p(int(host_ptr)) if host_ptr else None,
                                                    C.c_void_p(int(results_ptr)) if results_ptr else None))

    def lane_collect_preset_device(self, lane, slots, inst0, images_ptr, stride, n=None, results_ptr=0):
        """``collect_preset_device`` issued on a lane: uint8 [n, stride] slot images at ``images_ptr`` (stride >= the slot
        size; the tail of each row is left alone) and int32 [n] marks at ``results_ptr`` (optional).  ``slots`` is a scalar or
        [n]; it is read during the call."""
        sl = np.asarray(slots, np.uint8).reshape(-1)
        n = sl.size if n is None else int(n)
        sl = np.ascontiguousarray(np.broadcast_to(sl, (max(n, 0),)) if sl.size == 1 else sl)
        if sl.size != max(n, 0):
            raise ValueError("slots and n give different instance counts")
        _check(self._fn("lane_collect_preset_device")(self._h, int(lane), int(inst0), n, sl.ctypes.data_as(C.c_void_p),
                                                      C.c_void_p(int(images_ptr)) if images_ptr else None, C.c_size_t(int(stride)),
                                                      C.c_void_p(int(results_ptr)) if results_ptr else None))

    def lane_export_instances(self, lane, inst0, n, images_ptr, stride=None):
        """``export_instances`` issued on a lane: uint8 [n, stride] instance images at ``images_ptr`` (stride >=
        ``instance_image_size()``, its default; the tail of each row is left alone)."""
        stride = self.instance_image_size() if stride is None else int(stride)
        _check(self._fn("lane_export_instances")(self._h, int(lane), int(inst0), int(n), C.c_void_p(int(images_ptr)) if images_ptr else None,
                                                 C.c_size_t(stride)))

    def lane_response_device(self, lane, freqs, fs, inst0, n, out_ptr):
        """``response(freqs, fs, inst0, n, out_ptr)`` issued on a lane: complex64 [n, outputs, 2 inputs, n_freqs] at
        ``out_ptr``.  ``freqs`` is read during the call."""
        f = np.ascontiguousarray(freqs, np.float32).reshape(-1)
        _check(self._fn("lane_response_device")(self._h, int(lane), int(inst0), int(n), f.ctypes.data_as(C.c_void_p), f.size, C.c_float(fs),
                                                C.c_void_p(int(out_ptr)) if out_ptr else None))

    def lane_get_preset_mute(self, lane, inst0, n, states_ptr):
        """``get_preset_mute`` issued on a lane: PRESET_MUTE [n] at ``states_ptr``."""
        _check(self._fn("lane_get_preset_mute")(self._h, int(lane), int(inst0), int(n), C.c_void_p(int(states_ptr)) if states_ptr else None))

    def lane_get_spdif_tx(self, lane, inst0, n, tx_ptr):
        """``get_spdif_tx`` issued on a lane: SPDIF_TX [n] at ``tx_ptr``."""
        _check(self._fn("lane_get_spdif_tx")(self._h, int(lane), int(inst0), int(n), C.c_void_p(int(tx_ptr)) if tx_ptr else None))

    # Lane moves: a device moving into a lane's window, asynchronous on the lane streams; each returns without waiting.

    def lane_import_instances(self, lane, images, inst0):
        """``import_instances(images, inst0)`` issued on a lane ([inst0, inst0+n) inside its window): uint8 [n, stride]
        images in host memory, read during the call."""
        img = np.ascontiguousarray(images, np.uint8)
        if img.ndim != 2:
            raise ValueError("images must be [n, stride] bytes")
        _check(self._fn("lane_import_instances")(self._h, int(lane), int(inst0), int(img.shape[0]), img.ctypes.data_as(C.c_void_p),
                                                 C.c_size_t(img.shape[1])))

    def lane_copy_instances(self, src_lane, dst_lane, src, dst):
        """``copy_instances(src, dst)`` issued on lanes: every ``src[k]`` inside ``src_lane``'s window, every ``dst[k]``
        inside ``dst_lane``'s (the same lane repacks one group).  Ordered after the calls issued earlier on either lane;
        later calls on either lane run after it."""
        s, d = self._copy_lists(src, dst)
        _check(self._fn("lane_copy_instances")(self._h, int(src_lane), int(dst_lane), int(s.size), s.ctypes.data_as(C.c_void_p),
                                               d.ctypes.data_as(C.c_void_p)))


class ChainEngine(_ChainEngine):
    """Many independent DSPi device instances, whole signal chain (``dspi_chain_*``)."""
    _PRE, _PARAMS, _BIQUAD, _STATUS = "dspi_chain", L.CHAIN_PARAMS_F32, L.BIQUAD_F32, L.STATUS
    _ROLES, _OUTS, _PAIRS, _PLATFORM = L.CHAIN_EQ_CHANNELS, L.CHAIN_OUTPUTS, 4, L.PLATFORM_RP2350

    def __init__(self, arith, n_instances, max_frames, n_bands=L.NUM_BANDS, device=0):
        self.arith = ARITH[arith] if isinstance(arith, str) else int(arith)
        self.n_instances, self.max_frames, self.device = int(n_instances), int(max_frames), int(device)
        self._h = C.c_void_p()
        desc = _ChainDesc(self.arith, self.n_instances, int(n_bands), self.device, self.max_frames)
        _check(lib().dspi_chain_create(C.byref(self._h), C.byref(desc)))


def delay_samples(delay_ms, fs, is_last=False):
    return int(lib().dspi_delay_samples(delay_ms, fs, 1 if is_last else 0))


class _XfeedCfg(C.Structure):
    _fields_ = [("enabled", C.c_uint8), ("itd_enabled", C.c_uint8), ("preset", C.c_uint8), ("custom_fc", C.c_float), ("custom_feed_db", C.c_float)]


class _LevCfg(C.Structure):
    _fields_ = [("enabled", C.c_uint8), ("amount", C.c_float), ("speed", C.c_uint8), ("max_gain_db", C.c_float),
                ("lookahead", C.c_uint8), ("gate_threshold_db", C.c_float)]


def crossfeed_coefficients(fs, enabled=True, itd=True, preset=0, custom_fc=700.0, custom_feed_db=4.5):
    """``crossfeed_compute_coefficients`` -> XFEED_F32 record (state cleared)."""
    st = np.zeros(1, L.XFEED_F32)
    cfg = _XfeedCfg(int(enabled), int(itd), int(preset), custom_fc, custom_feed_db)
    lib().dspi_crossfeed_compute_coefficients_f32(st.ctypes.data, C.byref(cfg), fs)
    return st[0]


def leveller_coefficients(fs, amount=50.0, speed=0, max_gain_db=15.0, gate_db=-96.0):
    out = np.zeros(1, L.LEV_COEFFS)
    cfg = _LevCfg(1, amount, int(speed), max_gain_db, 1, gate_db)
    lib().dspi_leveller_compute_coefficients(out.ctypes.data, C.byref(cfg), fs)
    return out[0]


def loudness_table(fs, ref_spl=83.0, intensity_pct=100.0):
    t = np.zeros((L.LOUD_STEPS, 2), L.LOUD_F32)
    lib().dspi_loudness_compute_table_f32(t.ctypes.data, ref_spl, intensity_pct, fs)
    return t


def bulk_state_defaults(platform=L.PLATFORM_RP2350):
    """Power-on values of the globals ``bulk_params_apply`` edits (one ``BULK_STATE`` record)."""
    st = np.zeros(1, L.BULK_STATE)
    lib().dspi_bulk_state_defaults(st.ctypes.data_as(C.c_void_p), int(platform))
    return st


def bulk_params_apply(wire, state, exact_db=False):
    """``bulk_params_apply`` (bulk_params.c:178-377) on ``state`` (in place).  Returns the firmware's code: 0, -1 .. -4."""
    w = np.ascontiguousarray(wire).view(np.uint8).reshape(-1)
    assert w.size == L.WIRE_BULK.itemsize and state.dtype == L.BULK_STATE
    return int(lib().dspi_bulk_params_apply(w.ctypes.data_as(C.c_void_p), state.ctypes.data_as(C.c_void_p), int(bool(exact_db))))


def bulk_params_collect(state):
    """``bulk_params_collect`` (bulk_params.c:62-172): one ``WIRE_BULK`` record."""
    out = np.zeros(1, L.WIRE_BULK)
    lib().dspi_bulk_params_collect(state.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out


def bulk_state_to_chain(state, fs, host_volume_8_8=0, host_mute=False, biquads=None):
    """What the main loop derives after an apply: (chain params [1], biquads [1, roles, 12]) for the state's platform."""
    q28 = int(state["platform"][0]) == L.PLATFORM_RP2040
    P = np.zeros(1, L.CHAIN_PARAMS_Q28 if q28 else L.CHAIN_PARAMS_F32)
    roles = L.CHAINQ_EQ_CHANNELS if q28 else L.CHAIN_EQ_CHANNELS
    bq = np.zeros((1, roles, L.MAX_BANDS), L.BIQUAD_Q28 if q28 else L.BIQUAD_F32) if biquads is None else biquads
    fn = lib().dspi_bulk_state_to_chain_q28 if q28 else lib().dspi_bulk_state_to_chain_f32
    _check(fn(state.ctypes.data_as(C.c_void_p), C.c_float(fs), C.c_int16(int(host_volume_8_8)), int(bool(host_mute)),
              P.ctypes.data_as(C.c_void_p), bq.ctypes.data_as(C.c_void_p)))
    return P, bq


def preset_slot_size(platform=L.PLATFORM_RP2350):
    lib().dspi_preset_slot_size.restype = C.c_size_t
    return int(lib().dspi_preset_slot_size(int(platform)))


def crc32(data):
    lib().dspi_crc32.restype = C.c_uint32
    b = bytes(data)
    return int(lib().dspi_crc32(b, C.c_size_t(len(b))))


def preset_slot_collect(state, slot_index):
    """``collect_live_state`` (flash_storage.c:464-556): the slot image as bytes."""
    n = preset_slot_size(int(state["platform"][0]))
    out = np.zeros(n, np.uint8)
    _check(lib().dspi_preset_slot_collect(state.ctypes.data_as(C.c_void_p), int(slot_index), out.ctypes.data_as(C.c_void_p), C.c_size_t(n)))
    return out


def preset_slot_apply(image, slot_index, state, master_volume_mode=0, dir_master_volume_db=0.0):
    """The state part of ``preset_load`` on ``state`` (in place).  Returns 0 or 3 (PRESET_ERR_CRC)."""
    img = np.ascontiguousarray(image, np.uint8)
    return int(lib().dspi_preset_slot_apply(img.ctypes.data_as(C.c_void_p), C.c_size_t(img.size), int(slot_index), int(master_volume_mode),
                                           C.c_float(dir_master_volume_db), state.ctypes.data_as(C.c_void_p)))


SPDIF_CHANNEL_STATUS = bytes([0x04, 0x00, 0x00, 0x00, 0x0B])       # audio_spdif.c:82-88 (byte 3 = sample-rate code, set at run time)


def spdif_lookup_table():
    """The reference's 256-entry biphase-mark table (``audio_spdif.c:141-153``)."""
    t = np.zeros(256, np.uint32)
    lib().dspi_spdif_lookup_table(t.ctypes.data_as(C.c_void_p))
    return t


def spdif_encode_device(d_words, n_streams, frames, d_subframes, block_pos0=0, channel_status=SPDIF_CHANNEL_STATUS, device=0, stream=None):
    """Device pointers in/out: ``[n_streams][frames][2]`` int32 words -> ``[n_streams][frames][2][2]`` uint32 {l, h}."""
    cs = (C.c_uint8 * 5)(*channel_status)
    _check(lib().dspi_spdif_encode_device(int(device), C.c_void_p(int(d_words)), C.c_uint64(int(n_streams)), int(frames), int(block_pos0), cs,
                                          C.c_void_p(int(d_subframes)), C.c_void_p(int(stream) if stream else None)))


def spdif_encode_host(words, block_pos0=0, channel_status=SPDIF_CHANNEL_STATUS, device=0):
    """``words`` int32 ``[n_streams, frames, 2]`` (host) -> uint32 ``[n_streams, frames, 2, 2]`` ({l, h} per subframe)."""
    w = np.ascontiguousarray(words, np.int32)
    assert w.ndim == 3 and w.shape[2] == 2
    out = np.empty(w.shape + (2,), np.uint32)
    cs = (C.c_uint8 * 5)(*channel_status)
    _check(lib().dspi_spdif_encode_host(int(device), w.ctypes.data_as(C.c_void_p), C.c_uint64(w.shape[0]), int(w.shape[1]), int(block_pos0), cs,
                                        out.ctypes.data_as(C.c_void_p)))
    return out


def host_volume(volume_8_8):
    """``audio_set_volume``: returns (vol_mul as int16, loudness table row)."""
    idx = C.c_uint8()
    v = lib().dspi_host_volume(int(volume_8_8), C.byref(idx))
    return int(v), int(idx.value)


def preamp(db):
    """``update_preamp``: (linear float, Q28 int)."""
    lin, q = C.c_float(), C.c_int32()
    if lib().dspi_preamp(float(db), C.byref(lin), C.byref(q)) != 0:
        raise DspiError("preamp: NaN / Inf rejected")
    return lin.value, q.value


def master_volume(db):
    """``update_master_volume``: (linear float, Q15 int)."""
    lin, q = C.c_float(), C.c_int32()
    if lib().dspi_master_volume(float(db), C.byref(lin), C.byref(q)) != 0:
        raise DspiError("master volume: NaN / Inf rejected")
    return lin.value, q.value


class ChainEngineQ28(_ChainEngine):
    """Many independent RP2040-shape instances (2 in -> 5 out), Q28 arithmetic (``dspi_chainq_*``)."""
    _PRE, _PARAMS, _BIQUAD, _STATUS = "dspi_chainq", L.CHAIN_PARAMS_Q28, L.BIQUAD_Q28, L.STATUS_Q28
    _ROLES, _OUTS, _PAIRS, _PLATFORM = L.CHAINQ_EQ_CHANNELS, L.CHAINQ_OUTPUTS, 2, L.PLATFORM_RP2040

    def __init__(self, n_instances, max_frames, n_bands=L.NUM_BANDS, device=0):
        self.n_instances, self.max_frames, self.device = int(n_instances), int(max_frames), int(device)
        self._h = C.c_void_p()
        desc = _ChainDesc(ARITH_Q28, self.n_instances, int(n_bands), self.device, self.max_frames)
        _check(lib().dspi_chainq_create(C.byref(self._h), C.byref(desc)))


def crossfeed_coefficients_q28(fs, enabled=True, itd=True, preset=0, custom_fc=700.0, custom_feed_db=4.5):
    st = np.zeros(1, L.XFEED_Q28)
    cfg = _XfeedCfg(int(enabled), int(itd), int(preset), custom_fc, custom_feed_db)
    lib().dspi_crossfeed_compute_coefficients_q28(st.ctypes.data, C.byref(cfg), fs)
    return st[0]


def loudness_table_q28(fs, ref_spl=83.0, intensity_pct=100.0):
    t = np.zeros((L.LOUD_STEPS, 2), L.LOUD_Q28)
    lib().dspi_loudness_compute_table_q28(t.ctypes.data, ref_spl, intensity_pct, fs)
    return t
