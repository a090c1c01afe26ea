"""The plan of vb200_decode_streams_packets, restated in plain C (oracle/vb_oracle_decode_streams.c), against the
stock decoder's own vorbis_dsp_state after every vorbis_synthesis_blockin (oracle/ref_decode_plan.c), without a GPU:
the packet status and block flag, the samples pcmout returns, granulepos, pcm_returned, pcm_current, sequence and
sample_count of every packet, at full and half rate, on the seven kinds of stream of make_streams (a stream shorter
than a long block, a partial last packet, a non-audio packet, a truncated packet, a zero-byte packet, a packetno gap,
a beginning trim), with granulepos on every packet and on page-final packets only.  Cutting a stream's packets into
pieces with the state carried gives the same records.  make_streams also serves tests/test_gpu_decode_streams.py."""
import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode
from oracle import decode_streams as ds

CASES = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, -0.1)]
KINDS = ["short", "partial", "nonaudio", "truncated", "empty", "gap", "trim"]


def _need():
    if not (decode.available() and ds.ref_available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


_enc = {}


def make_streams(ch, rate, q, page_final=False):
    """the seven streams of one setup: (buf, hdr rows, [audio rows per stream]) with all streams' packets in buf.
    page_final: granulepos -1 except on every fourth packet and the last (as on Ogg pages)."""
    key = (ch, rate, q)
    if key not in _enc:
        _enc[key] = [decode.encode(ch, rate, q, probe_signal(ch, rate, secs, seed=900 + i))
                     for i, secs in enumerate((1000 / rate, 0.53, 0.41, 0.37, 0.33, 0.45, 0.5))]
    encs = _enc[key]
    bufs, audios, off = [], [], 0
    for kind, p in zip(KINDS, encs):
        a = p.audio.copy()
        m = len(a) // 2
        if kind == "nonaudio":                      # the comment header in the middle
            row = p.meta[1].copy()
            row[2], row[3], row[4] = -1, 0, a[m, 4]
            a = np.concatenate([a[:m], row[None], a[m:]])
        elif kind == "truncated":
            a[m, 1] //= 2
            a[m + 2, 1] = 1
        elif kind == "empty":
            a[m, 1] = 0
        elif kind == "gap":
            a = np.delete(a, m, axis=0)
        elif kind == "trim":                        # the first granulepos (packet 3) 700 samples behind the count
            a[:, 2] = np.where(a[:, 2] >= 0, a[:, 2] - 700, a[:, 2])
            a[:3, 2] = -1
        if page_final:
            keep = (np.arange(len(a)) % 4 == 3) | (np.arange(len(a)) == len(a) - 1)
            a[:, 2] = np.where(keep, a[:, 2], -1)
        a[:, 0] += off
        bufs.append(p.buf)
        audios.append(a)
        off += len(p.buf)
    return np.concatenate(bufs), encs[0].hdr, audios


@pytest.mark.parametrize("ch,rate,q", CASES)
@pytest.mark.parametrize("page_final", [False, True])
@pytest.mark.parametrize("half", [False, True])
def test_plan_equals_reference_state(ch, rate, q, page_final, half):
    _need()
    buf, hdr, audios = make_streams(ch, rate, q, page_final)
    bs = None
    seen = set()
    for kind, a in zip(KINDS, audios):
        pcm, ref, modebits = ds.ref_decode(buf, hdr, a, ch, halfrate=half)
        if bs is None:
            ident = buf[int(hdr[0, 0]):int(hdr[0, 0] + hdr[0, 1])]
            bs = [1 << int(ident[28] & 15), 1 << int(ident[28] >> 4)]
        plan = ds.Plan(bs, modebits, half)
        got = plan.run(buf, a)
        for k in range(len(a)):
            assert (got[k, :8] == ref[k]).all(), "%s packet %d: oracle %s reference %s" % (kind, k, got[k, :8], ref[k])
        assert got[:, 2].sum() == pcm.shape[1]
        seen.update(int(s) for s in ref[:, 0] if s)
        # a cut into pieces with the state carried gives the same records
        plan.restart()
        cuts = sorted(min(max(x, 0), len(a)) for x in (0, 1, 2, len(a) // 3, len(a) // 3, len(a) - 1, len(a)))
        pieces = np.concatenate([plan.run(buf, a[x:y]) for x, y in zip(cuts[:-1], cuts[1:])])
        assert (pieces == got).all(), kind
        if kind == "trim":
            assert got[3, 8] > 0, "no beginning trim"
        if kind == "partial" and not page_final:
            assert got[-1, 9] < got[-1, 10], "no end trim"
    assert seen == {-135}, seen                      # OV_ENOTAUDIO for the header packet and the empty one
