"""welle.io_b200 — GPU-native DAB/DAB+ physical-layer decode path (sm_90a / H100 CUDA behind a C ABI).

The directory name contains a dot, so import it by path (see tests/conftest.py::load_pkg or __graft_entry__.py):
    spec = importlib.util.spec_from_file_location("welle_io_b200", ".../welle.io_b200/__init__.py", submodule_search_locations=[...])
"""
from .dabb200 import (Context, Channelizer, DabbError, survey_candidates, CANDIDATE_DTYPE, DevBuf, build, load_library, LIB_PATH, EXPORTS, RESULT_DTYPE, TII_DTYPE, TII_MAX, BER_DTYPE, CLOCK_DTYPE, COMBINE_DTYPE, ACQ_DTYPE, MER_DTYPE, MER_GROUPS, MAX_BRANCHES,  # noqa: F401
                      FFT_EXACT, FFT_FMA, NCO_EXACT, NCO_FAST, DEMAP_REFERENCE, DEMAP_WEIGHTED, CLOCK_OFF, CLOCK_TRACK, ACQ_REFERENCE, ACQ_ROBUST, IQ_CF32, IQ_U8, IQ_S8, IQ_S16LE, IQ_S16BE, FRAME_DECODED, FRAME_NEED_SAMPLES, FRAME_NO_SYNC, FRAME_ACQUIRING,
                      L, K, TU, TS, TG, TNULL, TF, SOFT_PER_FRAME, MAX_SUBCH, Options,
                      PLACEMENT_THRESHOLD_BEFORE_PEAK, PLACEMENT_STRONGEST_PEAK, PLACEMENT_EARLIEST_PEAK_WITH_BINNING,
                      FREQSYNC_PATTERN_OF_ZEROS, FREQSYNC_GET_MIDDLE, FREQSYNC_CORRELATE_PRS)
from . import sharding  # noqa: F401
