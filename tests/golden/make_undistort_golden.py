"""TEST INFRASTRUCTURE: mints tests/golden/undistort_ref.npz, the reference's mve::image::image_undistort_k2k4<uint8_t>
on the seeded cases of tests/undistort_reference.py, through oracle/_ref/undistort_harness (built by oracle/undistort.mk
from the reference sources).  The photos are regenerated from their seeds; the file holds the results as
tests/undistort_reference.fixture_entries lays them out, written with fixed zip timestamps so that a second run gives
the same bytes.

    python tests/golden/make_undistort_golden.py"""
import io
import os
import subprocess
import sys
import tempfile
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from mve_b200 import synth                   # noqa: E402
from tests import undistort_reference as UR   # noqa: E402

HARNESS = os.path.join(ROOT, "oracle", "_ref", "undistort_harness")
OUT = os.path.join(ROOT, "tests", "golden", "undistort_ref.npz")


def main():
    cases = UR.cases()
    data = {}
    with tempfile.TemporaryDirectory(prefix="golden_") as tmp:
        args = []
        for k, (name, w, h, c, flen, k2, k4, seed) in enumerate(cases):
            fin, fout = os.path.join(tmp, "in%d.mvei" % k), os.path.join(tmp, "out%d.mvei" % k)
            synth.write_mvei(fin, UR.make_image(w, h, c, seed))
            args += [fin, fout, repr(flen), repr(k2), repr(k4)]
        subprocess.run([HARNESS] + args, check=True, capture_output=True)
        for k, case in enumerate(cases):
            data.update(UR.fixture_entries(case, synth.read_mvei(os.path.join(tmp, "out%d.mvei" % k))))
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for key in sorted(data):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(data[key]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)
    print("undistort", len(cases), "cases,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
