"""Writes tests/golden/sf_formats_v1.npz: the unmodified reference's answers (oracle.bind.Ref: RSDecoder::DecodeSuperframe and
SuperframeFilter::Feed) for every superframe of plainref.sf_all_inputs() - the four DAB+ audio formats at 1 .. 64 RS columns, chosen
error counts per column, headers that must not synchronise.  Plain arrays, nothing pickled: per case its name, SHA-256 of the input
(pins the seeded case generator) and of the corrected superframe, DecodeSuperframe's (corrected, uncorrectable), the filter's FECInfo
(uncorrectable, corrected) and its count of AUs whose CRC failed.  Needs the reference build (oracle/_ref/libwelle_ref.so):

    python tests/golden/make_sf_formats.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "sf_formats_v1.npz")


def record(ref):
    sys.path.insert(0, os.path.dirname(HERE))
    import plainref
    cases = plainref.sf_all_inputs()
    rows = []
    for name, sf in cases:
        out, corr, unc = ref.rs_decode_superframe(sf)
        fec, au_err, _ = ref.superframe_filter(sf.reshape(5, -1))
        assert len(fec) == 1, (name, fec)
        rows.append((hashlib.sha256(sf.tobytes()).digest(), hashlib.sha256(out.tobytes()).digest(), corr, unc, fec[0][0], fec[0][1], au_err))
    sha = lambda k: np.frombuffer(b"".join(r[k] for r in rows), np.uint8).reshape(-1, 32)
    col = lambda k: np.array([r[k] for r in rows], np.int32)
    return dict(name=np.array([c[0].encode() for c in cases]), input_sha256=sha(0), output_sha256=sha(1), rs_corr=col(2), rs_uncorr=col(3),
                fec_uncorr=col(4), fec_corr=col(5), au_errors=col(6))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle.bind import Ref
    assert Ref.available(), "build the reference first (WELLE_IO_SRC=<welle.io sources> python __graft_entry__.py)"
    np.savez_compressed(PATH, **record(Ref()))
    print("wrote", PATH)
