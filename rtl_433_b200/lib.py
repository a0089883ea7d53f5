"""ctypes binding of the C ABI in include/r433b.h (rtl_433_b200/csrc/libr433b.so).

Python is plumbing only: every sample is processed by the CUDA kernels inside the shared
library.  If the library is missing or no CUDA device is usable this module raises; there is
no CPU path.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.environ.get("R433B_LIB") or os.path.join(CSRC, "libr433b.so")  # override: tuning experiments only

FMT_CU8, FMT_CS16, FMT_CS8, FMT_CF32 = 2, 4, 0x102, 0x204
FPDM_CLASSIC, FPDM_MINMAX, FPDM_AUTO = 0, 1, 2
PACKAGE_OOK, PACKAGE_FSK = 1, 2

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-fmad=false",
              "-shared", "-Xcompiler", "-fPIC,-ffp-contract=off"]

EXPORTS = ["r433b_create", "r433b_destroy", "r433b_last_error", "r433b_set_levels", "r433b_set_fm_low_pass",
           "r433b_set_devices", "r433b_set_r_devices", "r433b_set_pipeline", "r433b_process", "r433b_fetch", "r433b_get_timing",
           "r433b_get_counts", "r433b_copy_stage", "r433b_event_to_bitbuffer", "r433b_package_to_pulse_data",
           "r433b_package_file_pos", "r433b_dispatch", "r433b_dispatch_r_devices", "r433b_stream_digest",
           "r433b_pulses_create", "r433b_pulses_destroy", "r433b_pulses_clear", "r433b_pulses_load_ook",
           "r433b_pulses_load_rfraw", "r433b_pulses_add", "r433b_pulses_count", "r433b_pulses_get", "r433b_process_pulses",
           "r433b_format_ook", "r433b_format_ook_header", "r433b_format_vcd", "r433b_format_vcd_header",
           "r433b_dump_logic_u8", "r433b_set_gates", "r433b_get_gated",
           "r433b_dispatch_r_devices_parallel", "r433b_analyze", "r433b_analysis_get", "r433b_analysis_text",
           "r433b_analysis_events", "r433b_submit", "r433b_wait", "r433b_grab_plan", "r433b_grab_copy", "r433b_grab_tail",
           "r433b_chain_create", "r433b_chain_destroy", "r433b_process_chained", "r433b_chain_base",
           "r433b_chain_grab", "r433b_set_split", "r433b_chain_split", "r433b_process_mixed",
           "r433b_process_mixed_chained"]


def build(force=False, verbose=False):
    """nvcc -> csrc/libr433b.so for sm_90a (cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, n) for n in sorted(os.listdir(CSRC)) if n.endswith((".cu", ".cuh", ".hpp"))]
    srcs += [os.path.join(os.path.dirname(HERE), "include", n) for n in ("r433b.h", "r433b_abi.h")]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH, os.path.join(CSRC, "r433b_api.cu")]
    subprocess.check_call(cmd)
    return LIB_PATH


class Device(C.Structure):
    _fields_ = [("modulation", C.c_uint32), ("short_width", C.c_float), ("long_width", C.c_float),
                ("reset_limit", C.c_float), ("gap_limit", C.c_float), ("sync_width", C.c_float),
                ("tolerance", C.c_float), ("priority", C.c_uint32)]


class Batch(C.Structure):
    _fields_ = [("data", C.c_void_p), ("offsets", C.POINTER(C.c_uint64)), ("n_streams", C.c_uint32),
                ("sample_format", C.c_uint32), ("samp_rate", C.c_uint32), ("center_frequency", C.c_uint32),
                ("fpdm_mode", C.c_uint32), ("block_bytes", C.c_uint32), ("data_on_device", C.c_int32),
                ("want_stages", C.c_int32), ("lengths", C.POINTER(C.c_uint64))]


class Package(C.Structure):
    _fields_ = [("stream", C.c_uint32), ("seq", C.c_uint32), ("type", C.c_int32), ("block", C.c_int32),
                ("offset", C.c_uint64), ("end_pos", C.c_uint64), ("start_ago", C.c_uint32), ("end_ago", C.c_uint32),
                ("num_pulses", C.c_uint32), ("pulse_off", C.c_uint32), ("pulse_count", C.c_uint32),
                ("ook_low_estimate", C.c_int32), ("ook_high_estimate", C.c_int32), ("fsk_f1_est", C.c_int32),
                ("fsk_f2_est", C.c_int32), ("first_pair", C.c_uint32)]


PACKAGE_DTYPE = np.dtype([("stream", "<u4"), ("seq", "<u4"), ("type", "<i4"), ("block", "<i4"), ("offset", "<u8"),
                          ("end_pos", "<u8"), ("start_ago", "<u4"), ("end_ago", "<u4"), ("num_pulses", "<u4"),
                          ("pulse_off", "<u4"), ("pulse_count", "<u4"), ("ook_low_estimate", "<i4"),
                          ("ook_high_estimate", "<i4"), ("fsk_f1_est", "<i4"), ("fsk_f2_est", "<i4"),
                          ("first_pair", "<u4")])
assert PACKAGE_DTYPE.itemsize == C.sizeof(Package) == 72

PAIR_DTYPE = np.dtype([("offset", "<u8"), ("bytes", "<u4"), ("events", "<u4"), ("gated_single", "<u4"), ("gated_multi", "<u4")])
assert PAIR_DTYPE.itemsize == 24


class Results(C.Structure):
    _fields_ = [("n_packages", C.c_uint32), ("n_devices", C.c_uint32), ("packages", C.c_void_p),
                ("pulse_pool", C.c_void_p), ("gap_pool", C.c_void_p), ("pairs", C.c_void_p), ("events", C.c_void_p),
                ("event_bytes", C.c_uint64), ("n_events", C.c_uint64), ("n_samples", C.c_uint64), ("n_gated", C.c_uint64)]


class HistBin(C.Structure):
    _fields_ = [("count", C.c_uint32), ("sum", C.c_int32), ("mean", C.c_int32), ("min", C.c_int32), ("max", C.c_int32)]


class Histogram(C.Structure):
    _fields_ = [("bins_count", C.c_uint32), ("bins", HistBin * 16)]


class Analysis(C.Structure):
    _fields_ = [("hist", Histogram * 5), ("total_period", C.c_int32)]


class Guess(C.Structure):
    _fields_ = [("modulation", C.c_uint32), ("short_width", C.c_float), ("long_width", C.c_float), ("reset_limit", C.c_float),
                ("gap_limit", C.c_float), ("sync_width", C.c_float), ("tolerance", C.c_float), ("last_gap", C.c_int32),
                ("sliced", C.c_int32)]


class Gate(C.Structure):
    _fields_ = [("min_bits", C.c_uint16), ("code_single", C.c_int8), ("code_multi", C.c_int8)]


class Timing(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("detect_ms", C.c_float), ("slice_ms", C.c_float), ("d2h_ms", C.c_float),
                ("total_ms", C.c_float), ("detect_launches", C.c_uint32), ("slice_launches", C.c_uint32),
                ("front_ms", C.c_float), ("front_launches", C.c_uint32), ("front_redone", C.c_uint32),
                ("front_repairs", C.c_uint32), ("idle_skipped", C.c_uint32), ("idle_rewalks", C.c_uint32),
                ("grab_ms", C.c_float), ("chain_folds", C.c_uint32), ("chain_fm_rebuilds", C.c_uint32),
                ("grab_ring_ms", C.c_float), ("split_segments", C.c_uint32), ("split_rewalks", C.c_uint32),
                ("split_rounds", C.c_uint32), ("split_merge_ms", C.c_float), ("mixed_classes", C.c_uint32),
                ("mixed_order_ms", C.c_float)]


class StreamFormat(C.Structure):
    _fields_ = [("sample_format", C.c_uint32), ("samp_rate", C.c_uint32), ("center_frequency", C.c_uint32)]


SPLIT_AUTO = 0xFFFFFFFF  # r433b_set_split: segment size chosen from the batch's shape

GRAB_ALL, GRAB_UNKNOWN, GRAB_KNOWN, GRAB_UNDECODED = 1, 2, 3, 4
GRAB_RING = 12 * 262144  # SIGNAL_GRABBER_BUFFER


class GrabRing(C.Structure):
    _fields_ = [("pushed", C.c_uint64), ("tail", C.c_void_p), ("counter", C.c_uint32)]


GRAB_DTYPE = np.dtype([("stream", "<u4"), ("first_package", "<u4"), ("n_packages", "<u4"), ("grab_len", "<u4"),
                       ("bytes", "<u4"), ("counter", "<u4"), ("run_end", "<i8")])
assert GRAB_DTYPE.itemsize == 32


class PulseData(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("sample_rate", C.c_uint32), ("depth_bits", C.c_uint), ("start_ago", C.c_uint),
                ("end_ago", C.c_uint), ("num_pulses", C.c_uint), ("pulse", C.c_int * 1200), ("gap", C.c_int * 1200),
                ("ook_low_estimate", C.c_int), ("ook_high_estimate", C.c_int), ("fsk_f1_est", C.c_int),
                ("fsk_f2_est", C.c_int), ("freq1_hz", C.c_float), ("freq2_hz", C.c_float), ("centerfreq_hz", C.c_float),
                ("range_db", C.c_float), ("rssi_db", C.c_float), ("snr_db", C.c_float), ("noise_db", C.c_float)]


assert C.sizeof(PulseData) == 9672

BITBUFFER_DTYPE = np.dtype([("num_rows", "<u2"), ("free_row", "<u2"), ("bits_per_row", "<u2", (50,)),
                            ("syncs_before_row", "<u2", (50,)), ("bb", "u1", (50, 128))])
assert BITBUFFER_DTYPE.itemsize == 6604

EVENT_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(PulseData), C.c_void_p)

_lib = None


def load():
    """dlopen the in-tree library; fails loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a). There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    L.r433b_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    L.r433b_destroy.argtypes = [C.c_void_p]
    L.r433b_last_error.restype = C.c_char_p
    L.r433b_last_error.argtypes = [C.c_void_p]
    L.r433b_set_levels.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float]
    L.r433b_set_fm_low_pass.argtypes = [C.c_void_p, C.c_float]
    L.r433b_set_pipeline.argtypes = [C.c_void_p, C.c_int]
    L.r433b_set_split.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.r433b_set_devices.argtypes = [C.c_void_p, C.POINTER(Device), C.c_uint32]
    L.r433b_set_r_devices.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.r433b_process.argtypes = [C.c_void_p, C.POINTER(Batch)]
    L.r433b_process_mixed.argtypes = [C.c_void_p, C.POINTER(Batch), C.POINTER(StreamFormat)]
    L.r433b_process_mixed_chained.argtypes = [C.c_void_p, C.POINTER(Batch), C.POINTER(StreamFormat), C.c_void_p, C.c_void_p]
    L.r433b_chain_create.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)]
    L.r433b_chain_destroy.argtypes = [C.c_void_p]
    L.r433b_process_chained.argtypes = [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p]
    L.r433b_chain_base.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64)]
    L.r433b_chain_grab.argtypes = [C.c_void_p, C.c_int]
    L.r433b_chain_split.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.r433b_fetch.argtypes = [C.c_void_p, C.POINTER(Results)]
    L.r433b_get_timing.argtypes = [C.c_void_p, C.POINTER(Timing)]
    L.r433b_get_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.r433b_stream_digest.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.POINTER(C.c_uint64)]
    L.r433b_copy_stage.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64]
    L.r433b_event_to_bitbuffer.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    L.r433b_package_to_pulse_data.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.POINTER(PulseData)]
    L.r433b_package_file_pos.restype = C.c_float
    L.r433b_package_file_pos.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32]
    L.r433b_dispatch.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, EVENT_FN, C.c_void_p]
    L.r433b_dispatch_r_devices.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.c_void_p, C.c_uint32]
    L.r433b_dispatch_r_devices_parallel.argtypes = [C.c_void_p, C.POINTER(Results), C.c_void_p, C.c_uint32, C.c_uint32]
    L.r433b_submit.argtypes = [C.c_void_p, C.POINTER(Batch)]
    L.r433b_wait.argtypes = [C.c_void_p, C.POINTER(Results)]
    L.r433b_analyze.argtypes = [C.c_void_p, C.POINTER(Results)]
    L.r433b_analysis_get.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.POINTER(Analysis), C.POINTER(Guess)]
    L.r433b_analysis_text.restype = C.c_size_t
    L.r433b_analysis_text.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.c_char_p, C.c_size_t]
    L.r433b_analysis_events.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint32),
                                        C.POINTER(C.c_uint32)]
    L.r433b_set_gates.argtypes = [C.c_void_p, C.POINTER(Gate), C.c_uint32]
    L.r433b_grab_plan.argtypes = [C.c_void_p, C.POINTER(Results), C.c_int, C.POINTER(GrabRing), C.POINTER(C.c_void_p),
                                  C.POINTER(C.c_uint32)]
    L.r433b_grab_copy.argtypes = [C.c_void_p, C.POINTER(Results), C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]
    L.r433b_grab_tail.argtypes = [C.c_void_p, C.POINTER(Results), C.c_void_p, C.POINTER(C.c_uint64)]
    L.r433b_get_gated.restype = C.c_uint64
    L.r433b_get_gated.argtypes = [C.c_void_p]
    L.r433b_pulses_create.restype = C.c_void_p
    L.r433b_pulses_destroy.argtypes = [C.c_void_p]
    L.r433b_pulses_clear.argtypes = [C.c_void_p]
    L.r433b_pulses_load_ook.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_size_t, C.c_uint32]
    L.r433b_pulses_load_rfraw.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p]
    L.r433b_pulses_add.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.r433b_pulses_count.restype = C.c_uint32
    L.r433b_pulses_count.argtypes = [C.c_void_p]
    L.r433b_pulses_get.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.r433b_process_pulses.argtypes = [C.c_void_p, C.c_void_p]
    for name in ("r433b_format_ook", "r433b_format_ook_header", "r433b_format_vcd", "r433b_format_vcd_header"):
        getattr(L, name).restype = C.c_size_t
    L.r433b_format_ook.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t]
    L.r433b_format_ook_header.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    L.r433b_format_vcd.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    L.r433b_format_vcd_header.argtypes = [C.c_uint32, C.c_char_p, C.c_char_p, C.c_size_t]
    L.r433b_dump_logic_u8.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint8]
    _lib = L
    return L


def default_device_table(include_disabled=False):
    """The reference's r_device table (rtl_433_b200/data/devices_25.12.json)."""
    with open(os.path.join(HERE, "data", "devices_25.12.json")) as f:
        devs = json.load(f)["devices"]
    return [d for d in devs if include_disabled or d["disabled"] == 0]


def default_gates(devs):
    """[(min_bits, code_single, code_multi)] for a device table: the length gates tools/probe_gates.py derived from
    the reference's decoders (rtl_433_b200/data/gates_25.12.json); devices without an entry get no gate."""
    with open(os.path.join(HERE, "data", "gates_25.12.json")) as f:
        g = json.load(f)["gates"]
    return [tuple(g.get(str(d.get("protocol_num", -1)), (0, 0, 0))) for d in devs]


class R433Error(RuntimeError):
    pass


PULSE_DATA_DTYPE = np.dtype([("offset", "<u8"), ("sample_rate", "<u4"), ("depth_bits", "<u4"), ("start_ago", "<u4"),
                             ("end_ago", "<u4"), ("num_pulses", "<u4"), ("pulse", "<i4", (1200,)), ("gap", "<i4", (1200,)),
                             ("ook_low_estimate", "<i4"), ("ook_high_estimate", "<i4"), ("fsk_f1_est", "<i4"),
                             ("fsk_f2_est", "<i4"), ("freq1_hz", "<f4"), ("freq2_hz", "<f4"), ("centerfreq_hz", "<f4"),
                             ("range_db", "<f4"), ("rssi_db", "<f4"), ("snr_db", "<f4"), ("noise_db", "<f4")], align=True)
assert PULSE_DATA_DTYPE.itemsize == 9672


def _as_pd_ptr(pd):
    """ctypes PulseData or numpy PULSE_DATA_DTYPE record -> (address, keep-alive object)."""
    if isinstance(pd, PulseData):
        return C.addressof(pd), pd
    a = np.ascontiguousarray(pd, dtype=PULSE_DATA_DTYPE).reshape(-1)[:1].copy()
    return a.ctypes.data, a


class Pulses:
    """A set of loaded packages (include/r433b.h: r433b_pulses): `.ook` text, RfRaw lines, pulse_data_t records.
    Host only; Context.process_pulses() runs the slicers on it."""

    def __init__(self):
        self.L = load()
        self.h = C.c_void_p(self.L.r433b_pulses_create())
        if not self.h:
            raise R433Error("r433b_pulses_create failed")

    def close(self):
        if self.h:
            self.L.r433b_pulses_destroy(self.h)
            self.h = None

    def clear(self):
        self.L.r433b_pulses_clear(self.h)

    def load_ook(self, text, samp_rate, stream=0):
        if isinstance(text, str):
            text = text.encode()
        n = self.L.r433b_pulses_load_ook(self.h, stream, text, len(text), samp_rate)
        if n < 0:
            raise R433Error(f"r433b_pulses_load_ook: {n}")
        return n

    def load_rfraw(self, line, stream=0):
        n = self.L.r433b_pulses_load_rfraw(self.h, stream, line.encode() if isinstance(line, str) else line)
        if n < 0:
            raise R433Error(f"r433b_pulses_load_rfraw: {n}")
        return n

    def add(self, pd, stream=0):
        ptr, _keep = _as_pd_ptr(pd)
        return self.L.r433b_pulses_add(self.h, stream, ptr)

    def __len__(self):
        return self.L.r433b_pulses_count(self.h)

    def get(self, i):
        out = np.zeros(1, PULSE_DATA_DTYPE)
        rc = self.L.r433b_pulses_get(self.h, i, out.ctypes.data)
        if rc:
            raise R433Error(f"r433b_pulses_get: {rc}")
        return out[0]


def format_ook(pd, received=None):
    """pulse_data_dump() text of a pulse_data_t (src/pulse_data.c:193-226)."""
    ptr, _keep = _as_pd_ptr(pd)
    buf = C.create_string_buffer(1 << 16)
    n = load().r433b_format_ook(ptr, received.encode() if received is not None else None, buf, len(buf))
    return buf.raw[:n].decode()


def format_vcd(pd, ch_id="'"):
    ptr, _keep = _as_pd_ptr(pd)
    buf = C.create_string_buffer(1 << 17)
    n = load().r433b_format_vcd(ptr, ord(ch_id), buf, len(buf))
    return buf.raw[:n].decode()


def format_vcd_header(sample_rate, date=""):
    buf = C.create_string_buffer(1024)
    n = load().r433b_format_vcd_header(sample_rate, date.encode(), buf, len(buf))
    return buf.raw[:n].decode()


def format_ook_header(created=None):
    buf = C.create_string_buffer(256)
    n = load().r433b_format_ook_header(created.encode() if created is not None else None, buf, len(buf))
    return buf.raw[:n].decode()


def dump_logic_u8(pd, length, buf_offset, bits):
    ptr, _keep = _as_pd_ptr(pd)
    out = np.zeros(length, np.uint8)
    load().r433b_dump_logic_u8(out.ctypes.data, length, buf_offset, ptr, bits)
    return out


class Chain:
    """Slots that carry each stream's demodulator state from one chained batch to the next (include/r433b.h:
    r433b_chain).  Pass it to Context.process(..., chain=, last=).  Context.close() closes the context's chains first;
    `with lib.Chain(ctx, n) as chain:` closes it at the end of the block."""

    def __init__(self, ctx, n_streams):
        self.L = ctx.L
        self.ctx = ctx
        self.n = n_streams
        h = C.c_void_p()
        ctx._check(self.L.r433b_chain_create(ctx.h, n_streams, C.byref(h)))
        self.h = h
        ctx._chains.append(self)

    def close(self):
        if self.h:
            self.L.r433b_chain_destroy(self.h)
            self.h = None
            self.ctx._chains.remove(self)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def base(self, stream):
        """Absolute sample index of the first sample of slot `stream`'s chunk in the last chained batch."""
        out = C.c_uint64()
        rc = self.L.r433b_chain_base(self.h, stream, C.byref(out))
        if rc:
            raise R433Error(f"r433b_chain_base: {rc}")
        return out.value

    def grab(self, mode):
        """Grab signals in `mode` (GRAB_*) on every slot, each its own run (include/r433b.h: r433b_chain_grab).  After
        each chained batch, ctx.grab_plan(mode) lists the grabs whose frames ended in it; ctx.grab_copy gathers them."""
        self.ctx._check(self.L.r433b_chain_grab(self.h, mode))

    def split(self, segment_blocks, warmup_blocks=1):
        """Segmented replay of this chain's batches (include/r433b.h: r433b_chain_split): each slot's chunk is walked in
        segments of segment_blocks blocks, the first from the carried state; 0 = off, SPLIT_AUTO = chosen from the
        batch.  Results are those of the unsplit chain; it may change between any two batches."""
        self.ctx._check(self.L.r433b_chain_split(self.h, segment_blocks, warmup_blocks))


class Context:
    """One GPU context (include/r433b.h: r433b_ctx)."""

    def __init__(self, cuda_device=0):
        self.L = load()
        h = C.c_void_p()
        rc = self.L.r433b_create(cuda_device, C.byref(h))
        if rc != 0:
            raise R433Error(f"r433b_create failed ({rc}): no usable CUDA device; there is no CPU fallback")
        self.h = h
        self._keep = None
        self.n_devices = 0
        self._chains = []

    def close(self):
        for chain in list(self._chains):
            chain.close()
        if self.h:
            self.L.r433b_destroy(self.h)
            self.h = None

    def _check(self, rc):
        if rc < 0:
            raise R433Error(f"r433b error {rc}: {self.L.r433b_last_error(self.h).decode()}")
        return rc

    def set_levels(self, use_mag_est=0, level_limit=0.0, min_level=-12.1442, min_snr=9.0):
        self._check(self.L.r433b_set_levels(self.h, use_mag_est, level_limit, min_level, min_snr))

    def set_fm_low_pass(self, v):
        self._check(self.L.r433b_set_fm_low_pass(self.h, v))

    def set_pipeline(self, groups):
        self._check(self.L.r433b_set_pipeline(self.h, groups))

    def set_split(self, segment_blocks, warmup_blocks=1):
        """Segmented replay of long streams (include/r433b.h: r433b_set_split) in process() and unchained
        process_mixed(): segment_blocks 0 = off, SPLIT_AUTO = chosen from the batch.  Results are those of the unsplit
        batch."""
        self._check(self.L.r433b_set_split(self.h, segment_blocks, warmup_blocks))

    def set_devices(self, devs):
        arr = (Device * len(devs))()
        for i, d in enumerate(devs):
            arr[i] = Device(d["modulation"], d["short_width"], d["long_width"], d["reset_limit"], d.get("gap_limit", 0.0),
                            d.get("sync_width", 0.0), d.get("tolerance", 0.0), d.get("priority", 0))
        self._check(self.L.r433b_set_devices(self.h, arr, len(devs)))
        self.n_devices = len(devs)

    def set_gates(self, gates):
        """gates: [(min_bits, code_single, code_multi)] per device, or None / [] to clear (include/r433b.h: r433b_gate)."""
        gates = gates or []
        arr = (Gate * max(1, len(gates)))()
        for i, g in enumerate(gates):
            arr[i] = Gate(*g)
        self._check(self.L.r433b_set_gates(self.h, arr, len(gates)))
        self.gates = list(gates)

    def gated(self):
        return int(self.L.r433b_get_gated(self.h))

    def process(self, data, offsets, sample_format, samp_rate=250000, center_frequency=433920000, fpdm_mode=FPDM_AUTO,
                block_bytes=0, data_on_device=False, want_stages=False, lengths=None, chain=None, last=None):
        """`data`: host numpy array (any dtype, contiguous) or an int device pointer.  With a Chain, stream i is the
        next chunk of slot i's file and `last[i]` says whether the file ends with it (r433b_process_chained)."""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        if isinstance(data, int):
            ptr = data
        else:
            data = np.ascontiguousarray(data)
            ptr = data.ctypes.data
        lens = None if lengths is None else np.ascontiguousarray(lengths, dtype=np.uint64)
        b = Batch(ptr, offs.ctypes.data_as(C.POINTER(C.c_uint64)), len(offs) - 1, sample_format, samp_rate,
                  center_frequency, fpdm_mode, block_bytes, int(data_on_device), int(want_stages),
                  None if lens is None else lens.ctypes.data_as(C.POINTER(C.c_uint64)))
        self._keep = (data, offs, lens)
        if chain is None:
            self._check(self.L.r433b_process(self.h, C.byref(b)))
            return
        flags = np.ascontiguousarray(np.ones(len(offs) - 1) if last is None else last, dtype=np.uint8)
        self._check(self.L.r433b_process_chained(self.h, C.byref(b), chain.h, flags.ctypes.data))

    def process_pulses(self, pulses):
        """All slicers on every package of a Pulses set (the slicer stage only); then fetch()/dispatch as usual."""
        self._keep = pulses
        self._check(self.L.r433b_process_pulses(self.h, pulses.h))

    def analyze(self):
        """The pulse analyzer (`rtl_433 -A`) on every package of the fetched batch."""
        self._check(self.L.r433b_analyze(self.h, C.byref(self._res)))

    def analysis(self, package_index):
        """-> (Analysis, Guess, text, [bitbuffer records of the trial demodulation])"""
        a, g = Analysis(), Guess()
        self._check(self.L.r433b_analysis_get(self.h, C.byref(self._res), package_index, C.byref(a), C.byref(g)))
        n = self.L.r433b_analysis_text(self.h, C.byref(self._res), package_index, None, 0)
        buf = C.create_string_buffer(n + 1)
        self.L.r433b_analysis_text(self.h, C.byref(self._res), package_index, buf, n + 1)
        ev, nb, ne = C.c_void_p(), C.c_uint32(), C.c_uint32()
        self._check(self.L.r433b_analysis_events(self.h, C.byref(self._res), package_index, C.byref(ev), C.byref(nb), C.byref(ne)))
        bbs = np.zeros(ne.value, BITBUFFER_DTYPE)
        at = 0
        for i in range(ne.value):
            used = C.c_uint32()
            rc = self.L.r433b_event_to_bitbuffer(ev.value + at, nb.value - at, 0, bbs[i:i + 1].ctypes.data, C.byref(used))
            if rc:
                raise R433Error("corrupt analyzer event stream")
            at += used.value
        return a, g, buf.value.decode(), bbs

    def process_mixed(self, data, offsets, formats, rates, freqs, lengths=None, fpdm_mode=FPDM_AUTO, data_on_device=False,
                      block_bytes=0, chain=None, last=None):
        """A batch whose stream i has its own sample format, rate and centre frequency (formats[i], rates[i], freqs[i];
        include/r433b.h: r433b_process_mixed).  `data`: host numpy array or an int device pointer.  With a Chain, stream
        i is the next chunk of slot i's file and `last[i]` says whether the file ends with it
        (r433b_process_mixed_chained).  Without a chain, set_split() splits the batch's long streams, every class in
        the same passes; a chain runs unsplit."""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offs) - 1
        if not (len(formats) == len(rates) == len(freqs) == n):
            raise ValueError("one format, rate and centre frequency per stream")
        if isinstance(data, int):
            ptr = data
        else:
            data = np.ascontiguousarray(data)
            ptr = data.ctypes.data
        lens = None if lengths is None else np.ascontiguousarray(lengths, dtype=np.uint64)
        fmt = (StreamFormat * max(1, n))()
        for i in range(n):
            fmt[i] = StreamFormat(int(formats[i]), int(rates[i]), int(freqs[i]))
        b = Batch(ptr, offs.ctypes.data_as(C.POINTER(C.c_uint64)), n, 0, 0, 0, fpdm_mode, block_bytes, int(data_on_device), 0,
                  None if lens is None else lens.ctypes.data_as(C.POINTER(C.c_uint64)))
        self._keep = (data, offs, lens)
        if chain is None:
            self._check(self.L.r433b_process_mixed(self.h, C.byref(b), fmt))
            return
        flags = np.ascontiguousarray(np.ones(n) if last is None else last, dtype=np.uint8)
        self._check(self.L.r433b_process_mixed_chained(self.h, C.byref(b), fmt, chain.h, flags.ctypes.data))

    def submit(self, data, offsets, sample_format, samp_rate=250000, center_frequency=433920000, fpdm_mode=FPDM_AUTO,
               block_bytes=0, data_on_device=False, lengths=None):
        """process() + fetch() on the context's worker thread; wait() returns what fetch() would."""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        if isinstance(data, int):
            ptr = data
        else:
            data = np.ascontiguousarray(data)
            ptr = data.ctypes.data
        lens = None if lengths is None else np.ascontiguousarray(lengths, dtype=np.uint64)
        b = Batch(ptr, offs.ctypes.data_as(C.POINTER(C.c_uint64)), len(offs) - 1, sample_format, samp_rate,
                  center_frequency, fpdm_mode, block_bytes, int(data_on_device), 0,
                  None if lens is None else lens.ctypes.data_as(C.POINTER(C.c_uint64)))
        self._keep = (data, offs, lens)
        self._check(self.L.r433b_submit(self.h, C.byref(b)))

    def wait(self):
        r = Results()
        self._check(self.L.r433b_wait(self.h, C.byref(r)))
        self._res = r
        return self._results_dict(r)

    def counts(self):
        out = (C.c_uint64 * 4)()
        self._check(self.L.r433b_get_counts(self.h, out))
        return {"packages": out[0], "events": out[1], "event_bytes": out[2], "samples": out[3]}

    def timing(self):
        t = Timing()
        self._check(self.L.r433b_get_timing(self.h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in Timing._fields_}

    def fetch(self):
        """-> dict of numpy views over the context's pinned host buffers."""
        r = Results()
        self._check(self.L.r433b_fetch(self.h, C.byref(r)))
        self._res = r
        return self._results_dict(r)

    @staticmethod
    def _results_dict(r):
        def view(ptr, nbytes, dtype):
            if not nbytes:
                return np.zeros(0, dtype)
            return np.frombuffer((C.c_uint8 * nbytes).from_address(ptr), dtype=dtype)

        npk = r.n_packages
        pk = view(r.packages, npk * 72, PACKAGE_DTYPE)
        pool_n = int((pk["pulse_off"].astype(np.int64) + pk["pulse_count"]).max()) if npk else 0
        return {"n_packages": npk, "n_devices": r.n_devices, "packages": pk,
                "pulse_pool": view(r.pulse_pool, pool_n * 4, np.int32), "gap_pool": view(r.gap_pool, pool_n * 4, np.int32),
                "pairs": view(r.pairs, npk * r.n_devices * 24, PAIR_DTYPE).reshape(npk, r.n_devices) if npk and r.n_devices else np.zeros((0, 0), PAIR_DTYPE),
                "events": view(r.events, r.event_bytes, np.uint8), "event_bytes": r.event_bytes, "n_events": r.n_events,
                "n_samples": r.n_samples, "n_gated": r.n_gated}

    def stream_digest(self, stream):
        """Position-independent checksum of everything the fetched batch holds for one stream."""
        out = C.c_uint64(0)
        self._check(self.L.r433b_stream_digest(self.h, C.byref(self._res), stream, C.byref(out)))
        return out.value

    def copy_stage(self, stream, n):
        am = np.zeros(n, np.int16)
        fm = np.zeros(n, np.int16)
        got = self._check(self.L.r433b_copy_stage(self.h, stream, am.ctypes.data, fm.ctypes.data, n))
        return am[:got], fm[:got]

    def grab_plan(self, mode, prior=None):
        """The signal grabber's files for the fetched batch (include/r433b.h: r433b_grab_plan) -> GRAB_DTYPE array.
        `prior` = (pushed, tail bytes, counter) of the run before this batch, or None when the batch starts it."""
        ring = None
        if prior is not None:
            pushed, tail, counter = prior
            tail = np.ascontiguousarray(tail, dtype=np.uint8)
            ring = GrabRing(pushed, tail.ctypes.data if tail.size else None, counter)
            self._grab_keep = tail
        ptr, n = C.c_void_p(), C.c_uint32()
        self._check(self.L.r433b_grab_plan(self.h, C.byref(self._res), mode, C.byref(ring) if ring is not None else None,
                                           C.byref(ptr), C.byref(n)))
        if not n.value:
            return np.zeros(0, GRAB_DTYPE)
        return np.frombuffer((C.c_uint8 * (n.value * GRAB_DTYPE.itemsize)).from_address(ptr.value), dtype=GRAB_DTYPE).copy()

    def grab_copy(self, first, count, nbytes):
        """The bytes of grabs [first, first + count) of the last plan, back to back (nbytes = their sum)."""
        out = np.zeros(max(int(nbytes), 1), np.uint8)
        self._check(self.L.r433b_grab_copy(self.h, C.byref(self._res), first, count, out.ctypes.data, int(nbytes)))
        return out[:int(nbytes)]

    def grab_tail(self):
        """-> (bytes pushed by the run after this batch, its last min(pushed, GRAB_RING) bytes): the next prior."""
        out = np.zeros(GRAB_RING, np.uint8)
        pushed = C.c_uint64()
        self._check(self.L.r433b_grab_tail(self.h, C.byref(self._res), out.ctypes.data, C.byref(pushed)))
        return pushed.value, out[:min(pushed.value, GRAB_RING)]

    def pulse_data(self, package_index):
        pd = PulseData()
        self._check(self.L.r433b_package_to_pulse_data(self.h, C.byref(self._res), package_index, C.byref(pd)))
        return pd

    def file_pos(self, package_index):
        return self.L.r433b_package_file_pos(self.h, C.byref(self._res), package_index)

    def dispatch(self, stream, fn):
        """fn(package_index, device_index, PulseData, bitbuffer numpy record) -> int"""
        def tramp(_user, pk, dv, pd, bits):
            bb = np.frombuffer((C.c_uint8 * 6604).from_address(bits), dtype=BITBUFFER_DTYPE)[0]
            return int(fn(pk, dv, pd.contents, bb) or 0)
        cb = EVENT_FN(tramp)
        self._check(self.L.r433b_dispatch(self.h, C.byref(self._res), stream, cb, None))

    def dispatch_native(self, stream, fn_ptr, user_ptr):
        """r433b_dispatch() with a native r433b_event_fn (address) and user pointer."""
        fn = C.cast(fn_ptr, EVENT_FN)
        self._check(self.L.r433b_dispatch(self.h, C.byref(self._res), stream, fn, user_ptr))

    def packages_of(self, stream):
        """Package dicts of one stream (integer header, float levels, widths) in order."""
        r = self._res
        npk = r.n_packages
        if not npk:
            return [], []
        pk = np.frombuffer((C.c_uint8 * (npk * 72)).from_address(r.packages), dtype=PACKAGE_DTYPE)
        pool_n = int((pk["pulse_off"].astype(np.int64) + pk["pulse_count"]).max())
        pp = np.frombuffer((C.c_uint8 * (pool_n * 4)).from_address(r.pulse_pool), dtype=np.int32)
        gp = np.frombuffer((C.c_uint8 * (pool_n * 4)).from_address(r.gap_pool), dtype=np.int32)
        out, index = [], []
        for gi in np.nonzero(pk["stream"] == stream)[0]:
            k = pk[gi]
            pd = self.pulse_data(int(gi))
            out.append({"type": int(k["type"]), "block": int(k["block"]), "offset": int(k["offset"]),
                        "sample_rate": pd.sample_rate, "depth_bits": pd.depth_bits, "start_ago": int(k["start_ago"]),
                        "end_ago": int(k["end_ago"]), "num_pulses": int(k["num_pulses"]),
                        "ook_low_estimate": int(k["ook_low_estimate"]), "ook_high_estimate": int(k["ook_high_estimate"]),
                        "fsk_f1_est": int(k["fsk_f1_est"]), "fsk_f2_est": int(k["fsk_f2_est"]),
                        "freq1_hz": pd.freq1_hz, "freq2_hz": pd.freq2_hz, "centerfreq_hz": pd.centerfreq_hz,
                        "range_db": pd.range_db, "rssi_db": pd.rssi_db, "snr_db": pd.snr_db, "noise_db": pd.noise_db,
                        "sample_file_pos": self.file_pos(int(gi)), "pulse_count": int(k["pulse_count"]),
                        "num_events": 0,
                        "pulse": pp[k["pulse_off"]:k["pulse_off"] + k["pulse_count"]].copy(),
                        "gap": gp[k["pulse_off"]:k["pulse_off"] + k["pulse_count"]].copy()})
            index.append(int(gi))
        return out, index
