"""Every device path on the 512/4096 block sizes that vorbisenc picks below q = 0 at 32-96 kHz and for low-rate
bitrate-managed encodes, and the generic-size transform instances (64, 128, 4096, 8192).  Bit-exact.

At these sizes the device runs code that the 256/2048 setups never launch: the generic `<0>` instances of
k_mdct_forward, k_mdct_backward and k_phaseA_transform (4096 and 8192 points, each thread striding over more
elements), the K = 16 instance of k_phaseA_psy3 (n = 2048), the generic k_phaseA_psy at n = 2048, and every buffer
that grows with n: the floor-1 fit's shared memory, twice the residue partitions, the half-rate decoder's <2048>
instances and a 106-step planner mark window.

The tests are the setup-family suite of tests/setup_families.py, on the rows of FAMILY:
- The stages against the oracle, which tests/test_oracle_vs_ref.py pins to the reference at (2, 44100, -0.1) and
  (6, 48000, -0.1) and tests/test_oracle_vs_ref.py::test_floor1_vs_reference at (2, 32000, -0.1).  The blocks the
  reference encoder cut are stored with its results under tests/golden/ref.
- Packets and PCM against the stock encoder and decoder (needs oracle/_ref).
- The generic sizes against the oracle bit for bit and against float64 direct formulas
  (tests/test_transform_fp64.py)."""
import pytest

import test_oracle_vs_ref as T
from setup_families import *  # noqa: F401,F403  (the suite's tests and fixtures)
from setup_families import (Family, gen_cfg, test_entropy_coder_fuzz, test_generic_size_halfrate,  # noqa: F401
                            test_generic_size_synthesis, test_generic_size_transforms,
                            test_generic_size_transforms_vs_fp64, test_stock_encoder_streams_in_pieces)

pytestmark = pytest.mark.gpu

LONG = [(2, 32000, -0.1), (2, 44100, -0.1), (6, 48000, -0.1)]
STOCK = [(2, 44100, -0.1), (1, 44100, -0.1), (6, 48000, -0.1)]        # where the stock encoder picks 512/4096
# name, channels, rate, max, nominal and min bitrate, and the small-reservoir settings: low-rate ABR, where
# vorbis_encode_setup_managed picks 512/4096
MANAGED = [("abr48", 2, 44100, -1, 48000, -1, None), ("mono32", 1, 44100, -1, 32000, -1, None)]


def check_long(setup, args):
    assert [setup.blocksize(0), setup.blocksize(1)] == [512, 4096]
    assert [setup.psy_n(k) for k in range(4)] == [256, 256, 2048, 2048]


FAMILY = Family(
    name="long", setups=LONG, capture={(2, 32000, -0.1): ("floor1", T.floor1_signal)}, check=check_long,
    blocksizes=lambda args: [512, 4096], nvec=[[1], [133], [4000]], fmts=[["f32"], ["s16"]],
    envelope=[[(2, 44100, -0.1)], [(6, 48000, -0.1)]],
    rows={"test_stock_encoder_packets": STOCK, "test_stock_managed_encoder": MANAGED, "test_stock_decoder": STOCK,
          "test_stock_halfrate_decoder": STOCK, "test_function_level_dropin": [(2, 44100, -0.1), (6, 48000, -0.1)]},
    fuzz=[(2, 44100, -0.1)])
