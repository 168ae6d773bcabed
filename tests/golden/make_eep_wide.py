"""Writes tests/golden/eep_wide_v1.npz: the unmodified reference's answers (oracle.bind.Ref: EEPProtection::deconvolve, then
EnergyDispersal::dedisperse) for every profile of plainref.eep_wide_profiles() it can decode - EEP-A and EEP-B from 200 kbit/s up to
1365 kbit/s (plainref.ref_decodes) - on the seeded softbits of plainref.eep_wide_soft.  Plain arrays, nothing pickled: per profile
(profile_a, bitrate, level), the SHA-256 of the input (pins the seeded generator) and of the output bits packed MSB first.  Needs the
reference build (oracle/_ref/libwelle_ref.so):

    python tests/golden/make_eep_wide.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "eep_wide_v1.npz")


def record(ref):
    sys.path.insert(0, os.path.dirname(HERE))
    import plainref
    profiles = [p for p in plainref.eep_wide_profiles() if plainref.ref_decodes(p[1])]
    ins, outs = [], []
    for pa, br, lv in profiles:
        soft = plainref.eep_wide_soft(pa, br, lv)
        bits = ref.eep_deconvolve(br, pa, lv, soft, True)
        ins.append(hashlib.sha256(soft.tobytes()).digest()); outs.append(hashlib.sha256(np.packbits(bits).tobytes()).digest())
    sha = lambda rows: np.frombuffer(b"".join(rows), np.uint8).reshape(-1, 32)
    return dict(profile=np.array(profiles, np.int32), input_sha256=sha(ins), output_sha256=sha(outs))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle.bind import Ref
    assert Ref.available(), "build the reference first (WELLE_IO_SRC=<welle.io sources> python __graft_entry__.py)"
    np.savez_compressed(PATH, **record(Ref()))
    print("wrote", PATH)
