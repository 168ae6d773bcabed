"""ctypes binding of libdab_b200.so (include/dab_b200.h) — the same C ABI a cgo/JNI/N-API stub would bind.

No computation happens in Python and there is no CPU fallback: if the shared library is missing or no CUDA device
is present, construction fails loudly.
"""
import ctypes as C
import os
import subprocess
import weakref

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DABB_LIB") or os.path.join(HERE, "libdab_b200.so")   # DABB_LIB: another build of the library, e.g. the parent's for scripts/gpu_ab.sh

L, K, TU, TS, TG, TNULL, TF = 76, 1536, 2048, 2552, 504, 2656, 196608
SOFT_PER_FRAME = 75 * 3072
MAX_SUBCH = 4
FFT_EXACT, FFT_FMA = 0, 1
NCO_EXACT, NCO_FAST = 0, 1
DEMAP_REFERENCE, DEMAP_WEIGHTED = 0, 1
CLOCK_OFF, CLOCK_TRACK = 0, 1
ACQ_REFERENCE, ACQ_ROBUST = 0, 1
IQ_CF32, IQ_U8, IQ_S8, IQ_S16LE, IQ_S16BE = 0, 1, 2, 3, 4
FRAME_DECODED, FRAME_NEED_SAMPLES, FRAME_NO_SYNC, FRAME_ACQUIRING = 0, 1, 2, 3


class DabbError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("n_streams", C.c_int32), ("transmission_mode", C.c_int32),
                ("fft_mode", C.c_int32), ("disable_coarse", C.c_int32), ("keep_taps", C.c_int32), ("n_subch_slots", C.c_int32),
                ("max_subch_cu", C.c_int32), ("ofdm_groups", C.c_int32), ("fft_placement", C.c_int32), ("freqsync_method", C.c_int32),
                ("nco_mode", C.c_int32), ("ofdm_tail_split", C.c_int32), ("reserved", C.c_int32 * 2)]


class Options(C.Structure):
    _fields_ = [("disable_coarse", C.c_int32), ("fft_placement", C.c_int32), ("freqsync_method", C.c_int32), ("decode_tii", C.c_int32), ("count_bit_errors", C.c_int32), ("reserved", C.c_int32 * 3)]
    # dabb_options.soft_demap is the C struct's former reserved[0]: the ctypes layout keeps the word inside `reserved`
    soft_demap = property(lambda self: self.reserved[0], lambda self, v: self.reserved.__setitem__(0, v))
    # dabb_options.sample_clock, the former reserved[1]
    sample_clock = property(lambda self: self.reserved[1], lambda self, v: self.reserved.__setitem__(1, v))
    # dabb_options.acquisition, the former reserved[2]
    acquisition = property(lambda self: self.reserved[2], lambda self, v: self.reserved.__setitem__(2, v))


PLACEMENT_THRESHOLD_BEFORE_PEAK, PLACEMENT_STRONGEST_PEAK, PLACEMENT_EARLIEST_PEAK_WITH_BINNING = 0, 1, 2
FREQSYNC_PATTERN_OF_ZEROS, FREQSYNC_GET_MIDDLE, FREQSYNC_CORRELATE_PRS = 0, 1, 2


class Subchannel(C.Structure):
    _fields_ = [("subch_id", C.c_int32), ("start_cu", C.c_int32), ("length_cu", C.c_int32), ("bitrate", C.c_int32),
                ("short_form", C.c_int32), ("uep_level", C.c_int32), ("eep_profile_a", C.c_int32), ("eep_level", C.c_int32),
                ("dabplus", C.c_int32)]


class FrameResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("start_index", C.c_int32), ("fine_corr", C.c_int32), ("coarse_corr", C.c_int32),
                ("snr_raw", C.c_int32), ("fib_crc_mask", C.c_int32), ("fic_ratio", C.c_int32),
                ("n_logical", C.c_int32 * MAX_SUBCH), ("n_rs_events", C.c_int32 * MAX_SUBCH), ("rs_uncorr_mask", C.c_int32 * MAX_SUBCH),
                ("rs_corr", (C.c_int32 * 4) * MAX_SUBCH), ("sf_ready", C.c_int32 * MAX_SUBCH), ("sf_au_count", C.c_int32 * MAX_SUBCH),
                ("sf_au_crc_mask", C.c_int32 * MAX_SUBCH), ("next_pos", C.c_int64), ("freq_corr_re", C.c_float), ("freq_corr_im", C.c_float),
                ("slevel", C.c_float), ("acq_failed", C.c_int32), ("reserved", C.c_int32 * 2)]


RESULT_DTYPE = np.dtype([("status", "<i4"), ("start_index", "<i4"), ("fine_corr", "<i4"), ("coarse_corr", "<i4"), ("snr_raw", "<i4"),
                         ("fib_crc_mask", "<i4"), ("fic_ratio", "<i4"), ("n_logical", "<i4", (4,)), ("n_rs_events", "<i4", (4,)),
                         ("rs_uncorr_mask", "<i4", (4,)), ("rs_corr", "<i4", (4, 4)), ("sf_ready", "<i4", (4,)), ("sf_au_count", "<i4", (4,)),
                         ("sf_au_crc_mask", "<i4", (4,)), ("next_pos", "<i8"), ("freq_corr_re", "<f4"), ("freq_corr_im", "<f4"),
                         ("slevel", "<f4"), ("acq_failed", "<i4"), ("reserved", "<i4", (2,))], align=True)
assert RESULT_DTYPE.itemsize == C.sizeof(FrameResult), (RESULT_DTYPE.itemsize, C.sizeof(FrameResult))

TII_MAX = 9
# dabb_tii_result: one stream's transmitter identification measurements of one step (tap 9)
TII_DTYPE = np.dtype([("count", "<i4"), ("evicted", "<i4"), ("skipped", "<i4"), ("reserved", "<i4"),
                      ("m", [("comb", "<i4"), ("pattern", "<i4"), ("delay_samples", "<i4"), ("error", "<f4")], (TII_MAX,))])
assert TII_DTYPE.itemsize == 16 + 16 * TII_MAX
# dabb_ber_result: one stream's channel bit errors of one step (tap 10)
BER_DTYPE = np.dtype([("fic_bits", "<i4"), ("fic_errors", "<i4"), ("fic_erasures", "<i4"), ("reserved", "<i4"),
                      ("subch", [("codewords", "<i4"), ("bits", "<i4"), ("errors", "<i4"), ("erasures", "<i4")], (MAX_SUBCH,))])
assert BER_DTYPE.itemsize == 80
# dabb_clock_result: one stream's sample-clock estimate of one step (tap 11)
CLOCK_DTYPE = np.dtype([("ppm", "<f4"), ("applied_ppm", "<f4"), ("frames", "<i4"), ("reserved", "<i4")])
assert CLOCK_DTYPE.itemsize == 16
# dabb_combine_result: one stream's diversity combination of one step (tap 12)
MAX_BRANCHES = 8
COMBINE_DTYPE = np.dtype([("members", "<i4"), ("mask", "<u4"), ("noise", "<f4"), ("reserved", "<i4")])
assert COMBINE_DTYPE.itemsize == 16
# dabb_acq_result: one stream's robust null search and phase reference excision of one step (tap 13)
ACQ_DTYPE = np.dtype([("searched", "<i4"), ("blocks", "<i4"), ("depth_db", "<f4"), ("excised", "<i4"), ("null_end", "<i8")])
assert ACQ_DTYPE.itemsize == 24
# dabb_mer_result: one stream's modulation error ratio of one step, over the band and per group of 24 carriers (tap 14)
MER_GROUPS = 64
MER_DTYPE = np.dtype([("points", "<i4"), ("mer_db", "<f4"), ("sig", "<i8"), ("err", "<i8"), ("group", [("sig", "<i4"), ("err", "<i4")], (MER_GROUPS,))])
assert MER_DTYPE.itemsize == 536


class IO(C.Structure):
    _fields_ = [("iq", C.c_void_p), ("iq_is_host", C.c_int32), ("stride_samples", C.c_int64), ("buf_start", C.c_void_p), ("buf_len", C.c_int64),
                ("results", C.c_void_p), ("fibs", C.c_void_p), ("msc", C.c_void_p), ("msc_stride", C.c_int32), ("sf", C.c_void_p), ("sf_stride", C.c_int32),
                ("iq_format", C.c_int32), ("carry_samples", C.c_int32)]


EXPORTS = ["dabb_create", "dabb_destroy", "dabb_last_error", "dabb_abi_version", "dabb_stream_reset", "dabb_set_options", "dabb_get_info", "dabb_select_subchannel",
           "dabb_remove_subchannel", "dabb_set_combining", "dabb_process", "dabb_process_async", "dabb_sync", "dabb_join_lanes", "dabb_submit", "dabb_collect", "dabb_cuda_stream", "dabb_kernel_launches",
           "dabb_read_tap", "dabb_profile", "dabb_profile_read", "dabb_ofdm_demod", "dabb_ofdm_demod_ex", "dabb_find_index", "dabb_find_index_ex", "dabb_coarse_estimate", "dabb_viterbi", "dabb_fic_decode", "dabb_msc_decode",
           "dabb_rs_superframes", "dabb_dev_alloc", "dabb_dev_free", "dabb_memcpy_h2d", "dabb_memcpy_d2h",
           "dabb_chan_create", "dabb_chan_destroy", "dabb_chan_input_range", "dabb_channelize", "dabb_survey", "dabb_survey_candidates", "dabb_set_mer"]


class ChanConfig(C.Structure):
    _fields_ = [("rate_hz", C.c_int64), ("iq_format", C.c_int32), ("n_inputs", C.c_int32), ("n_channels", C.c_int32), ("reserved", C.c_int32),
                ("input_of_channel", C.c_void_p), ("offset_hz", C.c_void_p)]


class ChanIO(C.Structure):
    _fields_ = [("in_", C.c_void_p), ("in_is_host", C.c_int32), ("in_stride", C.c_int64), ("in_start", C.c_void_p), ("in_len", C.c_int64),
                ("out", C.c_void_p), ("out_stride", C.c_int64), ("out_start", C.c_void_p), ("out_len", C.c_int64)]


class SurveyIO(C.Structure):
    _fields_ = [("in_", C.c_void_p), ("in_is_host", C.c_int32), ("iq_format", C.c_int32), ("in_stride", C.c_int64), ("n_inputs", C.c_int32),
                ("nfft", C.c_int32), ("in_len", C.c_int64), ("psd", C.c_void_p)]


# dabb_survey_candidate: one ensemble candidate of a spectrum
CANDIDATE_DTYPE = np.dtype([("offset_hz", "<i8"), ("score_db", "<f4"), ("reserved", "<i4")])


def survey_candidates(psd, rate_hz, min_score_db=6.0):
    """the ensemble candidates of one spectrum psd[nfft] (Context.survey) of an input at rate_hz (dabb_survey_candidates): a
    CANDIDATE_DTYPE array in ascending offset_hz"""
    lib = load_library()
    p = np.ascontiguousarray(psd, np.float32).reshape(-1)
    n = C.c_int32()
    cap = p.size // 2 + 1                       # runs of consecutive bins: never more than every other bin
    out = np.zeros(cap, CANDIDATE_DTYPE)
    rc = lib.dabb_survey_candidates(p.ctypes.data_as(C.c_void_p), C.c_int32(p.size), C.c_int64(int(rate_hz)), C.c_float(min_score_db),
                                    out.ctypes.data_as(C.c_void_p), C.c_int32(cap), C.byref(n))
    if rc != 0:
        raise DabbError(f"dabb_survey_candidates failed ({rc}): bad nfft ({p.size}) or rate ({rate_hz})")
    return out[:n.value]


def build():
    """Compile the CUDA sources for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(HERE, "csrc")])


def load_library():
    if not os.path.exists(LIB_PATH):
        raise DabbError(f"{LIB_PATH} is missing: run welle.io_b200.build() (nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    lib.dabb_last_error.restype = C.c_char_p
    lib.dabb_last_error.argtypes = [C.c_void_p]
    lib.dabb_cuda_stream.restype = C.c_void_p
    lib.dabb_cuda_stream.argtypes = [C.c_void_p]
    lib.dabb_kernel_launches.restype = C.c_int64
    lib.dabb_kernel_launches.argtypes = [C.c_void_p]
    lib.dabb_destroy.argtypes = [C.c_void_p]
    lib.dabb_destroy.restype = None
    lib.dabb_chan_destroy.argtypes = [C.c_void_p]
    lib.dabb_chan_destroy.restype = None
    return lib


def _addr(x):
    """integer address of a numpy array / torch tensor / DevBuf / raw int"""
    if isinstance(x, (int, np.integer)):
        return int(x)
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if hasattr(x, "ptr"):
        return x.ptr
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    raise TypeError(type(x))


def _vp(x):
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return x.ctypes.data_as(C.c_void_p)
    if isinstance(x, int):
        return C.c_void_p(x)
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    return x


class DevBuf:
    """Device memory owned through the ABI (so that tests need neither torch nor cuda-python)."""

    def __init__(self, ctx, nbytes):
        self.ctx, self.nbytes = ctx, int(nbytes)
        p = C.c_void_p()
        ctx._ck(ctx.lib.dabb_dev_alloc(ctx.h, C.c_size_t(self.nbytes), C.byref(p)))
        self.ptr = p.value

    def upload(self, arr):
        arr = np.ascontiguousarray(arr)
        assert arr.nbytes <= self.nbytes
        self.ctx._ck(self.ctx.lib.dabb_memcpy_h2d(self.ctx.h, C.c_void_p(self.ptr), _vp(arr), C.c_size_t(arr.nbytes)))
        return self

    def download(self, dtype, count=None):
        dt = np.dtype(dtype)
        n = self.nbytes // dt.itemsize if count is None else count
        out = np.empty(n, dt)
        self.ctx._ck(self.ctx.lib.dabb_memcpy_d2h(self.ctx.h, _vp(out), C.c_void_p(self.ptr), C.c_size_t(out.nbytes)))
        return out

    def free(self):
        if self.ptr:
            self.ctx.lib.dabb_dev_free(self.ctx.h, C.c_void_p(self.ptr))
            self.ptr = None


class Context:
    def __init__(self, n_streams=1, device=0, fft_mode=FFT_EXACT, disable_coarse=True, keep_taps=False, n_subch_slots=1,
                 max_subch_cu=0, ofdm_groups=0, fft_placement=0, freqsync_method=0, nco_mode=NCO_EXACT, ofdm_tail_split=0):
        self.lib = load_library()
        cfg = Config()
        cfg.abi_version = self.lib.dabb_abi_version()
        cfg.device, cfg.n_streams, cfg.transmission_mode = device, n_streams, 1
        cfg.fft_mode, cfg.disable_coarse, cfg.keep_taps = fft_mode, int(disable_coarse), int(keep_taps)
        cfg.n_subch_slots, cfg.max_subch_cu, cfg.ofdm_groups = n_subch_slots, max_subch_cu, ofdm_groups
        cfg.fft_placement, cfg.freqsync_method = int(fft_placement), int(freqsync_method)
        cfg.nco_mode, cfg.ofdm_tail_split = int(nco_mode), int(ofdm_tail_split)
        h = C.c_void_p()
        rc = self.lib.dabb_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise DabbError(f"dabb_create failed ({rc}): {self.lib.dabb_last_error(None).decode()}")
        self.h, self.n_streams, self.n_slots = h, n_streams, max(1, n_subch_slots)
        self._bufs = []
        self._chans = weakref.WeakSet()         # channelizers of this context: close() destroys them before the context

    def _ck(self, rc):
        if rc != 0:
            raise DabbError(f"libdab_b200 error {rc}: {self.lib.dabb_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            for ch in list(getattr(self, "_chans", ())):
                ch.destroy()
            self.lib.dabb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- memory helpers
    def dev(self, arr_or_bytes):
        if isinstance(arr_or_bytes, (int, np.integer)):
            return DevBuf(self, arr_or_bytes)
        a = np.ascontiguousarray(arr_or_bytes)
        return DevBuf(self, a.nbytes).upload(a)

    def cuda_stream(self):
        return self.lib.dabb_cuda_stream(self.h)

    def kernel_launches(self):
        return self.lib.dabb_kernel_launches(self.h)

    def sync(self):
        self._ck(self.lib.dabb_sync(self.h))

    def join_lanes(self):
        self._ck(self.lib.dabb_join_lanes(self.h))

    def profile(self, enable):
        self._ck(self.lib.dabb_profile(self.h, int(enable)))

    def profile_read(self):
        import json
        buf = C.create_string_buffer(16384)
        self._ck(self.lib.dabb_profile_read(self.h, buf, C.c_size_t(16384)))
        return json.loads(buf.value.decode())

    # ---- receiver control
    def reset(self, first=0, count=None, pos=0):
        self._ck(self.lib.dabb_stream_reset(self.h, first, self.n_streams if count is None else count, C.c_int64(pos)))

    def select_subchannel(self, start_cu, length_cu, bitrate, eep_profile_a=True, eep_level=3, short_form=False, uep_level=0,
                          dabplus=True, slot=0, first=0, count=None, subch_id=0):
        """streams [first, first + count) decode this sub-channel in `slot` (dabb_select_subchannel).  The streams of a slot are
        independent: each may have its own sub-channel, bitrate, protection and DAB/DAB+, and streams not named here decode on
        unchanged.  At most DABB_MAX_PROFILES (64) distinct protection profiles per context.  process() then needs msc_stride /
        sf_stride of at least the largest 3 x bitrate / 15 x bitrate among the streams selected in any slot."""
        sc = Subchannel(subch_id, start_cu, length_cu, bitrate, int(short_form), uep_level, int(eep_profile_a), eep_level, int(dabplus))
        self._ck(self.lib.dabb_select_subchannel(self.h, first, self.n_streams if count is None else count, slot, C.byref(sc)))

    def remove_subchannel(self, slot=0, first=0, count=None):
        """streams [first, first + count) stop decoding `slot`; the slot's other streams decode on unchanged"""
        self._ck(self.lib.dabb_remove_subchannel(self.h, first, self.n_streams if count is None else count, slot))

    def set_combining(self, leader=None):
        """diversity reception (dabb_set_combining): leader[s] == s for a stream that is alone or leads a group, else the stream whose
        group s joins (at most MAX_BRANCHES members per group, leader included); None dissolves every group.  Each leader's softbits
        become the demap of its group's noise-weighted differential products; every other member decodes on as it would alone."""
        if leader is None:
            self._ck(self.lib.dabb_set_combining(self.h, None, self.n_streams))
            return
        t = np.ascontiguousarray(leader, np.int32)
        self._ck(self.lib.dabb_set_combining(self.h, _vp(t), C.c_int32(t.size)))

    def set_mer(self, enable=True):
        """the modulation error ratio of every decoded frame's FIC softbits, over the band and in MER_GROUPS groups of 24 carriers
        (dabb_set_mer, tap 14), from the next step on"""
        self._ck(self.lib.dabb_set_mer(self.h, C.c_int32(int(bool(enable)))))

    def process(self, iq, stride, buf_start, buf_len, iq_is_host=False, msc_stride=0, sf_stride=0, want=("results", "fibs"), iq_format=0):
        S = self.n_streams
        bs = np.ascontiguousarray(buf_start, np.int64)
        assert bs.size == S
        io = IO()
        io.iq = _addr(iq)
        io.iq_is_host, io.stride_samples, io.buf_len = int(iq_is_host), stride, buf_len
        io.iq_format = iq_format
        io.buf_start = bs.ctypes.data
        out = {}
        if "results" in want:
            out["results"] = np.zeros(S, RESULT_DTYPE); io.results = out["results"].ctypes.data
        if "fibs" in want:
            out["fibs"] = np.zeros((S, 12, 32), np.uint8); io.fibs = out["fibs"].ctypes.data
        if msc_stride:
            out["msc"] = np.zeros((S, MAX_SUBCH, 4, msc_stride), np.uint8); io.msc = out["msc"].ctypes.data; io.msc_stride = msc_stride
        if sf_stride:
            out["sf"] = np.zeros((S, MAX_SUBCH, sf_stride), np.uint8); io.sf = out["sf"].ctypes.data; io.sf_stride = sf_stride
        self._ck(self.lib.dabb_process(self.h, C.byref(io)))
        return out

    def submit(self, iq, stride, buf_start, buf_len, msc_stride=0, sf_stride=0, want=("results", "fibs"), iq_format=0, out=None, carry=0):
        """pipelined host-buffer step (dabb_submit): returns immediately; collect() hands back the output dict of the oldest step.
        `out`: a dict returned by an earlier collect() to be reused for this step's results (saves allocating the arrays again).
        `carry`: the first `carry` samples of every window repeat the end of the previous submit's window and are not copied again"""
        S = self.n_streams
        bs = np.ascontiguousarray(buf_start, np.int64)
        io = IO()
        io.iq = _addr(iq)
        io.iq_is_host, io.stride_samples, io.buf_len, io.iq_format = 1, stride, buf_len, iq_format
        io.carry_samples = int(carry)
        io.buf_start = bs.ctypes.data
        if out is not None:
            io.results = out["results"].ctypes.data if "results" in out else None
            io.fibs = out["fibs"].ctypes.data if "fibs" in out else None
            if "msc" in out:
                io.msc = out["msc"].ctypes.data; io.msc_stride = out["msc"].shape[-1]
            if "sf" in out:
                io.sf = out["sf"].ctypes.data; io.sf_stride = out["sf"].shape[-1]
            self._ck(self.lib.dabb_submit(self.h, C.byref(io)))
            self._pending = getattr(self, "_pending", [])
            self._pending.append((out, bs, iq))
            return None
        out = {}
        if "results" in want:
            out["results"] = np.zeros(S, RESULT_DTYPE); io.results = out["results"].ctypes.data
        if "fibs" in want:
            out["fibs"] = np.zeros((S, 12, 32), np.uint8); io.fibs = out["fibs"].ctypes.data
        if msc_stride:
            out["msc"] = np.zeros((S, MAX_SUBCH, 4, msc_stride), np.uint8); io.msc = out["msc"].ctypes.data; io.msc_stride = msc_stride
        if sf_stride:
            out["sf"] = np.zeros((S, MAX_SUBCH, sf_stride), np.uint8); io.sf = out["sf"].ctypes.data; io.sf_stride = sf_stride
        self._ck(self.lib.dabb_submit(self.h, C.byref(io)))
        self._pending = getattr(self, "_pending", [])
        self._pending.append((out, bs, iq))          # keep the buffers alive until collected
        return None

    def collect(self):
        self._ck(self.lib.dabb_collect(self.h))
        out, _, _ = self._pending.pop(0)
        return out

    def process_async(self, iq_ptr, stride, buf_start, buf_len):
        bs = np.ascontiguousarray(buf_start, np.int64)
        io = IO()
        io.iq, io.iq_is_host, io.stride_samples, io.buf_len, io.buf_start = iq_ptr, 0, stride, buf_len, bs.ctypes.data
        self._ck(self.lib.dabb_process_async(self.h, C.byref(io)))

    def get_info(self, what):
        v = C.c_int64()
        self._ck(self.lib.dabb_get_info(self.h, int(what), C.byref(v)))
        return v.value

    def set_options(self, disable_coarse=True, fft_placement=0, freqsync_method=0, decode_tii=False, count_bit_errors=False, soft_demap=DEMAP_REFERENCE,
                    sample_clock=CLOCK_OFF, acquisition=ACQ_REFERENCE):
        """soft_demap: DEMAP_REFERENCE (the reference's demap) or DEMAP_WEIGHTED (weak carriers scaled by their level over the symbol's
        geometric-mean level, see dabb_options.soft_demap); sample_clock: CLOCK_OFF or CLOCK_TRACK (each stream's sample-clock error
        estimated from its frame timing and its phase ramp removed from the softbits, see dabb_options.sample_clock); acquisition:
        ACQ_REFERENCE (the reference's envelope-dip null search) or ACQ_ROBUST (the null found from the spectral level of 256-sample
        blocks, and narrowband interferers excised from the phase reference correlation, see dabb_options.acquisition)"""
        o = Options(); o.disable_coarse, o.fft_placement, o.freqsync_method, o.decode_tii = int(disable_coarse), int(fft_placement), int(freqsync_method), int(decode_tii)
        o.count_bit_errors, o.soft_demap, o.sample_clock = int(count_bit_errors), int(soft_demap), int(sample_clock)
        o.acquisition = int(acquisition)
        self._ck(self.lib.dabb_set_options(self.h, C.byref(o)))

    def read_tap(self, what, stride=0):
        """0 softbits, 1 CIR, 2 constellation points (75 x 16 per stream), 3 null symbol (2656 samples, NCO applied),
        4 TII spectra (PRS, null symbol), 5 frame results, 6 FIBs, 7 logical frames [S, MAX_SUBCH, 4, stride] and 8 superframes
        [S, MAX_SUBCH, stride] of the last step (also after process_async), 9 TII measurements (TII_DTYPE per stream), 10 channel bit
        errors (BER_DTYPE per stream), 11 sample-clock estimates (CLOCK_DTYPE per stream), 12 diversity combinations (COMBINE_DTYPE per
        stream), 13 robust acquisition (ACQ_DTYPE per stream), 14 modulation error ratio (MER_DTYPE per stream)"""
        if what == 7:
            out = np.zeros((self.n_streams, MAX_SUBCH, 4, stride), np.uint8)
        elif what == 8:
            out = np.zeros((self.n_streams, MAX_SUBCH, stride), np.uint8)
        elif what == 5:
            out = np.zeros(self.n_streams, RESULT_DTYPE)
        elif what == 6:
            out = np.zeros((self.n_streams, 12, 32), np.uint8)
        elif what == 0:
            out = np.zeros((self.n_streams, 75, 3072), np.int8)
        elif what == 2:
            out = np.zeros((self.n_streams, 75, 16), np.complex64)
        elif what == 3:
            out = np.zeros((self.n_streams, 2656), np.complex64)
        elif what == 4:
            out = np.zeros((self.n_streams, 2, 2048), np.complex64)
        elif what == 9:
            out = np.zeros(self.n_streams, TII_DTYPE)
        elif what == 10:
            out = np.zeros(self.n_streams, BER_DTYPE)
        elif what == 11:
            out = np.zeros(self.n_streams, CLOCK_DTYPE)
        elif what == 12:
            out = np.zeros(self.n_streams, COMBINE_DTYPE)
        elif what == 13:
            out = np.zeros(self.n_streams, ACQ_DTYPE)
        elif what == 14:
            out = np.zeros(self.n_streams, MER_DTYPE)
        else:
            out = np.zeros((self.n_streams, TU), np.float32)
        self._ck(self.lib.dabb_read_tap(self.h, what, _vp(out), C.c_size_t(out.nbytes)))
        return out

    def survey(self, x, nfft, in_len=None, iq_format=IQ_CF32, in_is_host=None):
        """the averaged power spectrum of every input (dabb_survey): a float32 array [n_inputs, nfft] whose bin j is at (j - nfft/2) R / nfft.
        x: a numpy array [n_inputs, samples] (or one input as a 1-d array; host, copied in the call; raw formats as bytes), or a
        DevBuf / device address of one input of in_len samples (in_is_host=False)"""
        if in_is_host is None:
            in_is_host = isinstance(x, np.ndarray)
        bps = (8, 2, 2, 4, 4)[iq_format] if 0 <= iq_format <= 4 else 1
        if isinstance(x, np.ndarray):
            xa = np.ascontiguousarray(x)
            rows = xa.reshape(1, -1) if xa.ndim == 1 else xa.reshape(xa.shape[0], -1)
            n_inputs, stride = rows.shape[0], rows[0].nbytes // bps
        else:
            if in_len is None:
                raise ValueError("Context.survey: device input needs in_len (its length in samples)")
            xa, n_inputs, stride = x, 1, int(in_len)
        in_len = stride if in_len is None else int(in_len)
        psd = np.zeros((n_inputs, int(nfft)), np.float32)
        io = SurveyIO(_addr(xa), int(bool(in_is_host)), int(iq_format), int(stride), n_inputs, int(nfft), in_len, psd.ctypes.data)
        self._ck(self.lib.dabb_survey(self.h, C.byref(io)))
        return psd

    # ---- stage-level (numpy in / numpy out; device staging through the ABI)
    def ofdm_demod(self, iq_frames, prs_start, nco=None, want_r1=False, want_fc=False, clock_ppm=None):
        """iq_frames: [n, stride] complex64; prs_start: [n] sample offsets of the first useful PRS sample; clock_ppm: None
        (dabb_ofdm_demod) or [n] float32 sample-clock ppm whose phase ramp each frame's demap removes (dabb_ofdm_demod_ex)"""
        iq = np.ascontiguousarray(iq_frames, np.complex64); n, stride = iq.shape
        d_iq = self.dev(iq); d_ps = self.dev(np.ascontiguousarray(prs_start, np.int64))
        d_soft = self.dev(n * SOFT_PER_FRAME)
        d_r1 = self.dev(n * 75 * K * 8) if want_r1 else None
        d_fc = self.dev(n * 8) if want_fc else None
        d_nco = self.dev(np.ascontiguousarray(nco, np.int32)) if nco is not None else None
        d_clk = self.dev(np.ascontiguousarray(clock_ppm, np.float32)) if clock_ppm is not None else None
        head = (self.h, C.c_void_p(d_iq.ptr), C.c_int64(stride), C.c_void_p(d_ps.ptr), n, C.c_void_p(d_nco.ptr) if d_nco else None)
        tail = (C.c_void_p(d_soft.ptr), C.c_void_p(d_r1.ptr) if d_r1 else None, C.c_void_p(d_fc.ptr) if d_fc else None)
        if d_clk is None:
            self._ck(self.lib.dabb_ofdm_demod(*head, *tail))
        else:
            self._ck(self.lib.dabb_ofdm_demod_ex(*head, C.c_void_p(d_clk.ptr), *tail))
        self.sync()
        out = [d_soft.download(np.int8).reshape(n, 75, 3072)]
        if want_r1:
            out.append(d_r1.download(np.complex64).reshape(n, 75, K))
        if want_fc:
            out.append(d_fc.download(np.complex64))
        for b in (d_iq, d_ps, d_soft, d_r1, d_fc, d_nco, d_clk):
            if b:
                b.free()
        return out[0] if len(out) == 1 else tuple(out)

    def coarse_estimate(self, iq_frames, prs_start, method=0):
        """OFDMProcessor::processPRS on aligned phase reference symbols; method = FREQSYNC_*"""
        iq = np.ascontiguousarray(iq_frames, np.complex64); n, stride = iq.shape
        d_iq = self.dev(iq); d_ps = self.dev(np.ascontiguousarray(prs_start, np.int64)); d_out = self.dev(4 * n)
        self._ck(self.lib.dabb_coarse_estimate(self.h, C.c_void_p(d_iq.ptr), C.c_int64(stride), C.c_void_p(d_ps.ptr), n, int(method), C.c_void_p(d_out.ptr)))
        self.sync()
        out = d_out.download(np.int32)
        for b in (d_iq, d_ps, d_out):
            b.free()
        return out

    def find_index(self, iq_frames, win_start, want_cir=False, placement=0):
        iq = np.ascontiguousarray(iq_frames, np.complex64); n, stride = iq.shape
        d_iq = self.dev(iq); d_ws = self.dev(np.ascontiguousarray(win_start, np.int64)); d_idx = self.dev(4 * n)
        d_cir = self.dev(4 * n * TU) if want_cir else None
        self._ck(self.lib.dabb_find_index_ex(self.h, C.c_void_p(d_iq.ptr), C.c_int64(stride), C.c_void_p(d_ws.ptr), n, int(placement), C.c_void_p(d_idx.ptr),
                                             C.c_void_p(d_cir.ptr) if d_cir else None))
        self.sync()
        idx = d_idx.download(np.int32)
        cir = d_cir.download(np.float32).reshape(n, TU) if want_cir else None
        for b in (d_iq, d_ws, d_idx, d_cir):
            if b:
                b.free()
        return (idx, cir) if want_cir else idx

    def viterbi(self, soft, nbits):
        soft = np.ascontiguousarray(soft, np.int8); n = soft.shape[0]
        assert soft.shape[1] == (nbits + 6) * 4
        d_s = self.dev(soft); d_o = self.dev(n * nbits)
        self._ck(self.lib.dabb_viterbi(self.h, C.c_void_p(d_s.ptr), n, nbits, C.c_void_p(d_o.ptr)))
        out = d_o.download(np.uint8).reshape(n, nbits)
        d_s.free(); d_o.free()
        return out

    def fic_decode(self, soft):
        soft = np.ascontiguousarray(soft, np.int8).reshape(-1, 9216); n = soft.shape[0]
        d_s = self.dev(soft); d_f = self.dev(n * 12 * 32); d_c = self.dev(4 * n)
        self._ck(self.lib.dabb_fic_decode(self.h, C.c_void_p(d_s.ptr), n, C.c_void_p(d_f.ptr), C.c_void_p(d_c.ptr)))
        fibs = d_f.download(np.uint8).reshape(n, 12, 32); crc = d_c.download(np.int32)
        for b in (d_s, d_f, d_c):
            b.free()
        return fibs, crc

    def msc_decode(self, soft, length_cu, bitrate, eep_profile_a=True, eep_level=3, short_form=False, uep_level=0):
        soft = np.ascontiguousarray(soft, np.int8).reshape(-1, length_cu * 64); n = soft.shape[0]
        sc = Subchannel(0, 0, length_cu, bitrate, int(short_form), uep_level, int(eep_profile_a), eep_level, 1)
        d_s = self.dev(soft); d_o = self.dev(n * 3 * bitrate)
        self._ck(self.lib.dabb_msc_decode(self.h, C.byref(sc), C.c_void_p(d_s.ptr), n, C.c_void_p(d_o.ptr)))
        out = d_o.download(np.uint8).reshape(n, 3 * bitrate)
        d_s.free(); d_o.free()
        return out

    def rs_superframes(self, sfs):
        sfs = np.ascontiguousarray(sfs, np.uint8); n, sf_len = sfs.shape
        d_s = self.dev(sfs); d_i = self.dev(16 * n)
        self._ck(self.lib.dabb_rs_superframes(self.h, C.c_void_p(d_s.ptr), n, sf_len, C.c_void_p(d_i.ptr)))
        self.sync()
        out = d_s.download(np.uint8).reshape(n, sf_len); info = d_i.download(np.int32).reshape(n, 4)
        d_s.free(); d_i.free()
        return out, info


class Channelizer:
    """Wideband channelizer of a context (dabb_chan_create): `offsets_hz[c]` is the centre of channel c in input
    `input_of_channel[c]` (default: all channels read input 0), every input at `rate_hz` in `iq_format` (IQ_*); `n_inputs` defaults to
    one more than the largest input a channel reads.  run() turns the inputs' samples into each channel's 2.048 Msps samples [out_start[c], out_start[c] + out_len) on the device, in a buffer that
    Context.process takes as its iq (stride = out_stride, buf_start = out_start).  Stateless: any range can be asked for at any time.
    destroy() (or the object's end) frees it and is safe to call twice; Context.close destroys the context's remaining channelizers
    first, so a channelizer never outlives its context."""

    def __init__(self, ctx, rate_hz, offsets_hz, input_of_channel=None, iq_format=IQ_CF32, n_inputs=None):
        self.ctx, self.lib = ctx, ctx.lib
        self.offsets = np.ascontiguousarray(offsets_hz, np.int64).reshape(-1)
        n = self.offsets.size
        self.input_of = np.ascontiguousarray(np.zeros(n, np.int32) if input_of_channel is None else input_of_channel, np.int32).reshape(-1)
        self.n_channels = n
        self.n_inputs = int(self.input_of.max()) + 1 if n_inputs is None and n else int(n_inputs or 1)
        self.rate_hz, self.iq_format = int(rate_hz), int(iq_format)
        cfg = ChanConfig(self.rate_hz, self.iq_format, self.n_inputs, n, 0, self.input_of.ctypes.data, self.offsets.ctypes.data)
        h = C.c_void_p()
        ctx._ck(self.lib.dabb_chan_create(ctx.h, C.byref(cfg), C.byref(h)))
        self.h = h
        ctx._chans.add(self)

    def input_range(self, out_start, out_len):
        """[first, end): the absolute input samples that outputs [out_start, out_start + out_len) of any channel read"""
        f, e = C.c_int64(), C.c_int64()
        self.ctx._ck(self.lib.dabb_chan_input_range(self.h, C.c_int64(int(out_start)), C.c_int64(int(out_len)), C.byref(f), C.byref(e)))
        return f.value, e.value

    def run(self, x, in_start, in_len, out_start, out_len, in_stride=None, in_is_host=None, out=None, out_stride=None):
        """x: the inputs, [n_inputs, in_stride] samples (numpy: host, copied in the call; DevBuf / int address: device) whose first
        samples are the absolute indices in_start[i].  out_start: one absolute output index per channel (an int: the same for all).
        Returns the device buffer (float2 [n_channels][out_stride]); `out` reuses one."""
        if in_is_host is None:
            in_is_host = isinstance(x, np.ndarray)
        if in_stride is None:           # a numpy array [n_inputs, ...]: one row per input
            in_stride = x.reshape(self.n_inputs, -1)[0].nbytes // (8, 2, 2, 4, 4)[self.iq_format]
        ins = np.ascontiguousarray(np.broadcast_to(np.asarray(in_start, np.int64), (self.n_inputs,)))
        outs = np.ascontiguousarray(np.broadcast_to(np.asarray(out_start, np.int64), (self.n_channels,)))
        out_stride = int(out_len if out_stride is None else out_stride)
        if out is None:
            out = self.ctx.dev(self.n_channels * out_stride * 8)
        xa = np.ascontiguousarray(x) if isinstance(x, np.ndarray) else None
        io = ChanIO(_addr(xa if xa is not None else x), int(bool(in_is_host)), int(in_stride), ins.ctypes.data, int(in_len),
                    _addr(out), out_stride, outs.ctypes.data, int(out_len))
        self.ctx._ck(self.lib.dabb_channelize(self.h, C.byref(io)))
        return out

    def destroy(self):
        if getattr(self, "h", None):
            self.lib.dabb_chan_destroy(self.h)
            self.ctx._chans.discard(self)
        self.h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass
