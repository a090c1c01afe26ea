"""k_floor1_fit through vb200_floor1_fit_dev against the CPU oracle, on every fixture's floors, with rows that
start 16-byte aligned (the fit quantises four lines per load) and rows that do not (one line per load)."""
import numpy as np
import pytest

from conftest import CONFIG_NAMES, load_setup
from vorbis_b200 import abi, lib as vlib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("W", [0, 1])
@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_floor1_fit_dev_row_alignment(oracle_lib, cuda_ok, name, W, offset):
    import torch
    setup = load_setup(name)
    ctx, o = vlib.Context(setup), oracle_lib.Oracle(setup)
    n, rows = setup.blocksize(W) // 2, 16 * setup.channels
    rng = np.random.default_rng(900 + W)
    logmask = rng.uniform(-140, 0, (rows, n)).astype(np.float32)
    logmdct = (logmask + rng.normal(0, 12, (rows, n))).astype(np.float32)
    logmask[0] = -200.0                                  # dBquant clips at 0: NULL fit
    want_posts, want_nz = o.floor1_fit(W, logmdct, logmask)
    assert (want_nz == 0).any() and (want_nz == 1).any()

    dev = torch.device("cuda", 0)
    buf = torch.zeros(2 * rows * n + 8, dtype=torch.float32, device=dev)
    d_mdct = buf[offset:offset + rows * n]              # offset 1: every row is 4-byte aligned only
    d_mask = buf[offset + rows * n + 4:offset + 2 * rows * n + 4]
    d_mdct.copy_(torch.from_numpy(logmdct.ravel()))
    d_mask.copy_(torch.from_numpy(logmask.ravel()))
    posts = torch.full((rows, abi.FLOOR1_STRIDE), -1, dtype=torch.int32, device=dev)
    nz = torch.full((rows,), -1, dtype=torch.int32, device=dev)
    ctx.floor1_fit_dev(W, rows, d_mdct.data_ptr(), d_mask.data_ptr(), posts.data_ptr(), nz.data_ptr())
    torch.cuda.synchronize()
    got_posts, got_nz = posts.cpu().numpy(), nz.cpu().numpy()
    assert np.array_equal(got_nz, want_nz), "fit_nonzero"
    assert np.array_equal(got_posts, want_posts), "posts: %d diffs" % (got_posts != want_posts).sum()
