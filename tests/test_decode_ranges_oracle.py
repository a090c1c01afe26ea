"""The premise of vb200_decode_ranges, on the reference itself and without a GPU: a range of a stream's output needs
only the blocks that finish its samples and the one decoded block before them.  On four setups (the last one
512/4096), the seven kinds of stream of make_streams (a stream shorter than a long block, a partial last packet, a
non-audio packet, a truncated packet, a zero-byte packet, a packetno gap, a beginning trim), granulepos on every
packet and on page-final packets only, full and half rate:
- oracle/decode_ranges.py's restatement of the plan gives the lengths, per-packet samples, granulepos, status and
  windows of oracle/vb_oracle_decode_streams.c (itself pinned to the reference's state by
  tests/test_decode_streams_oracle.py);
- for seeded requests, the stock decoder fed only the planned packets (priming block first), with granulepos -1 and
  e_o_s 0 so that it trims nothing, returns every finished sample of each block after the first; cut by the plan's
  windows these equal the slice of the stock decoder's whole-stream PCM, bit for bit."""
import numpy as np
import pytest

from oracle import decode
from oracle import decode_ranges as dr
from oracle import decode_streams as ds
from test_decode_streams_oracle import CASES, KINDS, make_streams


def _need():
    if not (decode.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def requests(length, packets, blks, rng, n=6):
    """seeded (start, length) pairs on a stream of `length` samples: the start, inside the first returned block,
    across the middle packet (where make_streams puts each kind's special packet), across every block that returns
    fewer samples than it finishes (the trims), the end, past it, and random ones"""
    out = [(0, 1500), (max(length - 1500, 0), 1500), (max(length - 300, 0), 1000), (length, 100), (10, 0)]
    first = next((b for b in blks if b["hi"] > b["lo"]), None)
    if first is not None:
        out.append((first["pos"] + 5, 700))
    out.append((max(int(packets[len(packets) // 2, 0]) - 900, 0), 2000))
    out += [(max(b["pos"] - 900, 0), 2000) for b in blks[1:] if b["hi"] - b["lo"] < b["fin"]]
    for _ in range(n):
        out.append((int(rng.integers(0, max(length, 1))), int(rng.integers(1, 6000))))
    return out


@pytest.mark.parametrize("ch,rate,q", CASES)
@pytest.mark.parametrize("page_final", [False, True])
@pytest.mark.parametrize("half", [False, True])
def test_range_plan_on_the_stock_decoder(ch, rate, q, page_final, half):
    _need()
    buf, hdr, audios = make_streams(ch, rate, q, page_final)
    rng = np.random.default_rng(rate + ch + page_final + 2 * half)
    ident = buf[int(hdr[0, 0]):int(hdr[0, 0] + hdr[0, 1])]
    bs = [1 << int(ident[28] & 15), 1 << int(ident[28] >> 4)]
    checked = 0
    for kind, a in zip(KINDS, audios):
        whole, ref, modebits = ds.ref_decode(buf, hdr, a, ch, halfrate=half)
        length, packets, blks = dr.blocks(buf, a, bs, modebits, half)
        # the restatement's bookkeeping is the oracle plan's
        rec = ds.Plan(bs, modebits, half).run(buf, a)
        assert length == whole.shape[1] == rec[:, 2].sum(), kind
        assert (packets[:, 3] == rec[:, 0]).all() and (packets[:, 2] == rec[:, 2]).all(), kind
        assert (packets[:, 1] == rec[:, 3]).all(), kind
        assert (packets[:, 0] == np.cumsum(rec[:, 2]) - rec[:, 2]).all(), kind
        dec = rec[:, 0] == 0
        assert [b["lo"] for b in blks] == list(rec[dec, 8]) and [b["hi"] for b in blks] == list(rec[dec, 9]), kind
        for start, n in requests(length, packets, blks, rng):
            got, kept = dr.plan(blks, start, n)
            assert got == min(n, max(0, length - start)), (kind, start, n)
            if not kept:
                assert got == 0
                continue
            rows = np.array([a[b["k"]] for b in kept], np.int64)
            rows[:, 2], rows[:, 3] = -1, 0                  # the stock decoder trims nothing
            pcm, r, _ = ds.ref_decode(buf, hdr, rows, ch, halfrate=half)
            assert r[0, 2] == 0
            fin = np.cumsum(r[:, 2]) - r[:, 2]
            out = np.zeros((ch, got), np.float32)
            for i, b in enumerate(kept[1:], 1):
                lo, hi = b["keep"]
                assert hi <= r[i, 2]
                out[:, b["at"]:b["at"] + hi - lo] = pcm[:, fin[i] + lo:fin[i] + hi]
            want = whole[:, start:start + got]
            assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), (kind, start, n)
            checked += 1
    assert checked > 40
