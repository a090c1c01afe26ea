"""The managed multi-stream driver (vb200ms_open_managed in vorbis_b200/host/vb200_mapping0.c): N bitrate-managed
encoders whose ready blocks go to the device together, one vb200_encode_dsp_managed call per block size and round,
the 15 packet blobs of every block written by the reference's own floor1_encode / residue backend, each stream's
bitrate manager choosing among them.  Every stream's packets (count, bytes, hash of all bytes in order) must equal
what the stock reference encoder of the same configuration produces for that stream alone.  Needs oracle/_ref (built
where the reference sources exist; the libraries travel)."""
import numpy as np
import pytest

from conftest import probe_signal

pytestmark = pytest.mark.gpu


def _signals(ch, rate, ns, secs):
    from test_plan_vs_ref import burst_signal
    n = int(rate * secs)
    sig = [probe_signal(ch, rate, secs, seed=40 + i)[:, :n] if i % 2 == 0 else burst_signal(ch, rate, secs, 50 + i)[:, :n]
           for i in range(ns)]
    return np.ascontiguousarray(np.stack(sig), np.float32)


@pytest.mark.parametrize("ch,rate,max_br,nominal,min_br", [(2, 44100, -1, 128000, -1), (1, 44100, -1, 64000, -1),
                                                           (2, 44100, 144000, -1, 112000)])
def test_managed_multistream_packets_identical(cuda_ok, ch, rate, max_br, nominal, min_br):
    from oracle import managed
    if not managed.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ns = 7
    pcm = _signals(ch, rate, ns, 0.8)
    blocks, rounds, launches, got = managed.ms_encode(ch, rate, max_br, nominal, min_br, pcm)
    total = 0
    for i in range(ns):
        nb, c, b, h = managed.stock_summary(ch, rate, max_br, nominal, min_br, pcm[i])
        assert got[i][:2] == (c, b), "stream %d: %d packets / %d bytes, stock %d / %d" % (i, got[i][0], got[i][1], c, b)
        assert got[i][2] == h, "stream %d packet bytes differ" % i
        assert c > 10
        total += nb
    assert blocks == total
    # a round takes at most one block per stream, and the streams drift apart around short-block runs; on average
    # several streams share each round's device calls.  The device work of a round does not grow with the stream
    # count: the envelope search of every stream, then one managed chain per block size (~15 kernels each)
    assert rounds * 2 <= blocks, "%d rounds for %d blocks: the streams' blocks are not batched" % (rounds, blocks)
    assert launches <= 30 * rounds, "%d launches in %d rounds" % (launches, rounds)


def test_managed_multistream_launches_independent_of_stream_count(cuda_ok):
    """the same 2 streams alone and among 12: launches per round stay within the same bound"""
    from oracle import managed
    if not managed.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ch, rate = 2, 44100
    pcm = _signals(ch, rate, 12, 0.5)
    per_round = []
    for ns in (2, 12):
        blocks, rounds, launches, got = managed.ms_encode(ch, rate, -1, 128000, -1, pcm[:ns])
        assert blocks > 0 and rounds > 0
        per_round.append(launches / rounds)
        for i in range(2):
            _, c, b, h = managed.stock_summary(ch, rate, -1, 128000, -1, pcm[i])
            assert got[i] == (c, b, h), "stream %d of %d differs from the stock encoder" % (i, ns)
    assert per_round[1] <= 1.25 * per_round[0] + 2, "launches per round: %.1f with 2 streams, %.1f with 12" % tuple(per_round)
