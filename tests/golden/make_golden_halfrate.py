#!/usr/bin/env python
"""Record the reference's half-rate decode (vorbis_synthesis_halfrate(vi, 1)) for tests/test_halfrate_oracle.py
and tests/test_gpu_halfrate.py into tests/golden/ref/halfrate/halfrate.npz, keys "<cfg>__<name>".  For every decode
fixture tests/golden/decode_<cfg>.npz: the block flags of its window, the half-rate PCM those blocks finish and
the two half windows of the halved block sizes.  Needs oracle/_ref/libvorbis_ref_halfrate.so (oracle/Makefile
builds it from the unmodified reference sources).  Writes no other file.

usage:  python tests/golden/make_golden_halfrate.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__  # noqa: E402
from conftest import CONFIG_NAMES  # noqa: E402
from oracle import halfrate  # noqa: E402
from test_halfrate_oracle import FIXTURE, reference_halfrate  # noqa: E402


def main():
    __graft_entry__.build()
    if not halfrate.ref_available():
        sys.exit("oracle/_ref/libvorbis_ref_halfrate.so is missing: it needs the reference sources")
    out = {}
    for name in CONFIG_NAMES:
        rec = reference_halfrate(name)
        out.update({"%s__%s" % (name, k): v for k, v in rec.items()})
        print(name, "blocks", len(rec["W"]), "pcm", rec["pcm"].shape)
    os.makedirs(os.path.dirname(FIXTURE), exist_ok=True)
    np.savez_compressed(FIXTURE, **out)


if __name__ == "__main__":
    main()
