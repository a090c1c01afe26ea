"""The multi-stream decode driver (vorbis_b200/host/vb200_decode.c, vb200md_*): 7 streams of one codec setup, of
different lengths, fed on a seeded schedule of 0-5 packets per stream per round, decode to the stock decoder's
vorbis_synthesis_pcmout sequence bit for bit (float) and to examples/decoder_example.c's int16 of it.  Among the
streams: one shorter than a long block, one whose last packet is partial (end trim by granulepos), one with a
non-audio packet in the middle.  vb200md_restart and re-feeding a stream reproduces its PCM, and the device launches
of a round stay bounded (two decode kernels) whatever the number of streams."""
import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode

pytestmark = pytest.mark.gpu

CASES = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2)]


def _streams(ch, rate, q):
    """7 encoded streams: (buf, audio meta, header meta) each"""
    out = []
    lengths = [0.9, 0.1, 1.3, 0.55, 0.7, 1.1, 0.4]
    for i, secs in enumerate(lengths):
        pcm = probe_signal(ch, rate, secs, seed=100 + i)
        if i == 1:
            pcm = pcm[:, :1000]                                # shorter than a long block
        if i == 3:
            pcm = pcm[:, :pcm.shape[1] - 333]                  # the last packet is partial
        p = decode.encode(ch, rate, q, pcm)
        audio = p.audio
        if i == 4:                                             # a non-audio packet (the comment header) mid-stream
            k = len(audio) // 2
            audio = np.concatenate([audio[:k], p.meta[1:2], audio[k:]])
        out.append((p, audio))
    return out


def _check_case(ch, rate, q, s16):
    enc = _streams(ch, rate, q)
    want = [decode.stock_decode(p, audio, ch, s16=s16) for p, audio in enc]
    assert want[1].shape[0 if s16 else 1] < 2048
    joined = decode.join([(p.buf, a, p.meta[:3]) for p, a in enc])
    rng = np.random.default_rng(ch * 1000 + int(q * 10))
    sched = rng.integers(0, 6, (400, len(enc)))
    got, st = decode.md_run(joined, sched, ch, s16=s16, restart=2)
    for s in range(len(enc)):
        assert got[s].shape == want[s].shape, "stream %d: %s vs %s" % (s, got[s].shape, want[s].shape)
        if s16:
            assert np.array_equal(got[s], want[s]), "stream %d int16" % s
        else:
            assert np.array_equal(got[s].view(np.uint32), want[s].view(np.uint32)), "stream %d float" % s
    assert np.array_equal(got[len(enc)].view(np.uint8), got[2].view(np.uint8)), "restart + re-feed"
    assert st["max_launches_per_round"] <= 2
    return want, st


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_driver_float_equals_stock_pcmout(cuda_ok, ch, rate, q):
    if not decode.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    _check_case(ch, rate, q, False)


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_driver_int16_equals_decoder_example(cuda_ok, ch, rate, q):
    if not decode.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    want, _ = _check_case(ch, rate, q, True)
    f = [decode.stock_decode(p, a, ch) for p, a in _streams(ch, rate, q)]
    for s in range(len(f)):
        conv = np.clip(np.floor(f[s] * np.float32(32767.0) + np.float32(0.5)), -32768, 32767).astype(np.int16).T
        assert np.array_equal(conv, want[s])


def test_driver_launches_do_not_grow_with_streams(cuda_ok):
    if not decode.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    p = decode.encode(2, 44100, 0.5, probe_signal(2, 44100, 0.6, seed=7))
    per_round = {}
    for ns in (2, 12):
        joined = decode.join([(p.buf, p.audio, p.meta[:3])] * ns)
        sched = np.full((10, ns), 3)
        _, st = decode.md_run(joined, sched, 2, keep=False)
        assert st["rounds"] > 1
        per_round[ns] = st["max_launches_per_round"]
    assert per_round[2] == per_round[12] == 2
