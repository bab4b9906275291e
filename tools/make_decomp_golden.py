"""Records the host decomposition (fq_ellipsoid_decomp) of tests/decomp_cases.py into tests/golden/decomp_host.npz:
face_ofs and Ab of every case, concatenated (case_ofs / row_ofs index them).  tests/test_pair_decomp_cpu.py compares the
library's output with it bit for bit, so a change to the host arithmetic shows.  Usage: python tools/make_decomp_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from faster_b200 import capi  # noqa: E402
import decomp_cases as dc  # noqa: E402


def main():
    names, face_ofs, Ab, case_ofs, row_ofs = [], [], [], [0], [0]
    for name, path, obs, r in dc.all_cases():
        polys = capi.ellipsoid_decomp(path, obs, dc.BBOX, r, dc.Z_GROUND, cap_rows=8192)
        fo = np.concatenate([[0], np.cumsum([len(b) for _, b in polys])]).astype(np.int32)
        names.append(name)
        face_ofs.append(fo)
        Ab.append(np.vstack([np.hstack([A, b[:, None]]) for A, b in polys]))
        case_ofs.append(case_ofs[-1] + len(fo))
        row_ofs.append(row_ofs[-1] + int(fo[-1]))
    out = os.path.join(ROOT, "tests", "golden", "decomp_host.npz")
    np.savez_compressed(out, names=np.array(names), face_ofs=np.concatenate(face_ofs), Ab=np.vstack(Ab),
                        case_ofs=np.asarray(case_ofs, np.int64), row_ofs=np.asarray(row_ofs, np.int64))
    print("wrote %s: %d cases, %d rows" % (out, len(names), row_ofs[-1]))


if __name__ == "__main__":
    main()
