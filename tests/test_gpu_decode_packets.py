"""Packets decoded on the device (vb200_decode_entropy, vb200_decode_packets_resume and the multi-stream decode
driver's device path) against the reference's own floor1_inverse1 and residue inverse:
- the staging (residue vectors as uint32, floor posts, presence) of every audio packet of seeded streams of five
  setups and of one bitrate-managed stream equals the reference's;
- so does the staging of packets cut at every byte length, and of packets with seeded bit flips after the header;
- vb200_decode_packets_resume equals vb200_decode_entropy + vb200_decode_dsp_resume bit for bit, in float and int16,
  at full and half rate, for streams cut into calls in several ways, in two launches per call; _dev equals the host
  form; bad arguments give VB200_EINVAL;
- the driver takes the device path for its three setups and decodes like the stock decoder on it and on the forced
  host path, also for a stream with truncated packets in the middle."""
import numpy as np
import pytest

from conftest import probe_signal
from oracle import decode
from oracle import decode_packets as dp
from vorbis_b200 import lib

pytestmark = pytest.mark.gpu

CASES = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2), (2, 44100, 0.1), (2, 32000, 0.0)]
DRIVER_CASES = [(2, 44100, 0.5), (1, 22050, 0.3), (6, 48000, 0.2)]
HEADER_BITS = 4                        # 1 + modebits (1 for two modes) + 2 for a long block


def _need():
    if not (decode.available() and dp.available()):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


_enc = {}


def _streams(ch, rate, q):
    """3 seeded encodings of one setup"""
    key = (ch, rate, q)
    if key not in _enc:
        _enc[key] = [decode.encode(ch, rate, q, probe_signal(ch, rate, secs, seed=300 + i))
                     for i, secs in enumerate((0.8, 0.45, 1.1))]
    return _enc[key]


def _pkts(p):
    return [bytes(p.buf[int(o):int(o + n)]) for o, n in p.audio[:, :2]]


def _check(p, drv, pkts, what):
    W = dp.ref_headers(p, pkts)
    ref = dp.ref_staging(p, pkts, W, drv.bs, drv.channels)
    got = dp.dev_staging(drv.ctx, pkts, W, drv.bs, drv.channels)
    assert np.array_equal(ref[0].view(np.uint32), got[0].view(np.uint32)), what + ": residue"
    assert np.array_equal(ref[1], got[1]), what + ": posts"
    assert np.array_equal(ref[2], got[2]), what + ": present"
    return W, ref


@pytest.fixture
def driver():
    made = []

    def make(p):
        d = dp.Driver(p)
        made.append(d)
        return d
    yield make
    for d in made:
        d.close()


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_stage_parity(cuda_ok, driver, ch, rate, q):
    _need()
    for i, p in enumerate(_streams(ch, rate, q)):
        drv = driver(p)
        assert drv.on_device
        W, ref = _check(p, drv, _pkts(p), "stream %d" % i)
        assert (W >= 0).all() and (W == 0).any() and (W == 1).any()
        assert ref[2].any()


def test_stage_parity_managed(cuda_ok, driver):
    _need()
    p = dp.encode_managed(2, 44100, probe_signal(2, 44100, 1.0, seed=11), nominal_br=128000)
    drv = driver(p)
    assert drv.on_device
    _check(p, drv, _pkts(p), "managed")


def _pick(W, n, rng):
    """n packet indices, both block sizes"""
    short, long_ = np.nonzero(W == 0)[0], np.nonzero(W == 1)[0]
    k = min(len(long_), n // 2)
    return np.concatenate([rng.choice(short, min(len(short), n - k), replace=False),
                           rng.choice(long_, k, replace=False)])


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_truncated_packets(cuda_ok, driver, ch, rate, q):
    _need()
    p = _streams(ch, rate, q)[0]
    drv = driver(p)
    pkts = _pkts(p)
    rng = np.random.default_rng(int(rate + 10 * ch + 100 * q))
    cut = [pkts[i][:k] for i in _pick(dp.ref_headers(p, pkts), 20, rng) for k in range(len(pkts[i]) + 1)]
    W, ref = _check(p, drv, cut, "truncated")
    assert (W < 0).any() and (W >= 0).any()
    assert (ref[2] == 0).any() and (ref[2] == 1).any()


@pytest.mark.parametrize("ch,rate,q", CASES)
def test_damaged_packets(cuda_ok, driver, ch, rate, q):
    _need()
    p = _streams(ch, rate, q)[1]
    drv = driver(p)
    pkts = _pkts(p)
    rng = np.random.default_rng(int(7 * rate + ch + 1000 * q))
    out = []
    for i in _pick(dp.ref_headers(p, pkts), 40, rng):
        a = np.frombuffer(pkts[i], np.uint8)
        nbits = 8 * len(a)
        if nbits <= HEADER_BITS:
            continue
        for _ in range(5):
            b = a.copy()
            for bit in rng.integers(HEADER_BITS, nbits, rng.integers(1, 9)):
                b[bit >> 3] ^= np.uint8(1 << (bit & 7))
            out.append(b.tobytes())
    _check(p, drv, out, "damaged")


def _pieces(nmax, how):
    if how == "one":
        return [(0, nmax)]
    if how == "two":
        return [(0, nmax // 3), (nmax // 3, nmax)]
    if how == "three":
        return [(0, 2), (2, nmax // 2 + 1), (nmax // 2 + 1, nmax)]
    return [(k, k + 1) for k in range(nmax)]


def _fused_case(drv, streams, how, s16, half):
    ctx, ch, bs = drv.ctx, drv.channels, drv.bs
    allp = [_pkts(p) for p in streams]
    Ws = [dp.ref_headers(streams[s], allp[s]) for s in range(len(streams))]
    flat = [b for pk in allp for b in pk]
    data = np.frombuffer(b"".join(flat) + b"\0", np.uint8).copy()
    starts = np.cumsum([0] + [len(b) for b in flat])
    first = np.cumsum([0] + [len(pk) for pk in allp])
    ns, nmax = len(streams), max(len(pk) for pk in allp)
    ka, kb = ctx.new_decode_carry(ns), ctx.new_decode_carry(ns)
    for a, b in _pieces(nmax, how):
        nblk = b - a
        count = np.array([max(0, min(len(allp[s]), b) - a) for s in range(ns)], np.int32)
        Wseq = np.zeros((ns, nblk), np.int32)
        pkt_off = np.zeros((ns, nblk), np.int64)
        pkt_bytes = np.zeros((ns, nblk), np.int32)
        for s in range(ns):
            for k in range(count[s]):
                Wseq[s, k] = Ws[s][a + k]
                g = first[s] + a + k
                pkt_off[s, k], pkt_bytes[s, k] = starts[g], starts[g + 1] - starts[g]
        coef_off, pcm_off, coef_len, pcm_len = lib.synthesis_layout(Wseq, bs, ch, halfrate=half, carry_W=ka[1],
                                                                    count=count)
        stride = max(pcm_len, 1)
        m = (np.arange(nblk)[None, :] < count[:, None]).reshape(-1)
        res, posts, present = ctx.decode_entropy(Wseq.reshape(-1)[m], pkt_off.reshape(-1)[m],
                                                 pkt_bytes.reshape(-1)[m], data, coef_off.reshape(-1)[m],
                                                 max(coef_len, 1))
        P = np.zeros((ns * nblk, ch, dp.FLOOR1_STRIDE), np.int32)
        Z = np.zeros((ns * nblk, ch), np.int32)
        P[m], Z[m] = posts, present
        want = ctx.decode_dsp_resume(Wseq, coef_off, res, P.reshape(ns, nblk, ch, -1), Z.reshape(ns, nblk, ch),
                                     pcm_off, stride, ka, count=count, s16=s16)
        l0 = ctx.launch_count()
        got = ctx.decode_packets_resume(Wseq, coef_off, max(coef_len, 1), pkt_off, pkt_bytes, data, pcm_off, stride,
                                        kb, count=count, s16=s16)
        assert ctx.launch_count() - l0 == 2
        assert np.array_equal(want.view(np.uint8), got.view(np.uint8)), "pcm, pieces %s, call at %d" % (how, a)
        assert np.array_equal(ka[0].view(np.uint32), kb[0].view(np.uint32)) and np.array_equal(ka[1], kb[1])


@pytest.mark.parametrize("ch,rate,q", DRIVER_CASES)
@pytest.mark.parametrize("how", ["one", "two", "three", "each"])
def test_fused_equals_entropy_then_dsp(cuda_ok, driver, ch, rate, q, how):
    _need()
    streams = _streams(ch, rate, q)[:2]
    drv = driver(streams[0])
    for half in (False, True):
        drv.ctx.synthesis_halfrate(half)
        for s16 in (False, True):
            _fused_case(drv, streams, how, s16, half)
    drv.ctx.synthesis_halfrate(False)


def test_fused_dev_equals_host_and_rejects_bad_arguments(cuda_ok, driver):
    _need()
    import torch
    p = _streams(2, 44100, 0.5)[0]
    drv = driver(p)
    ctx, ch, bs = drv.ctx, drv.channels, drv.bs
    pk = _pkts(p)[:12]
    W = dp.ref_headers(p, pk)
    data = np.frombuffer(b"".join(pk) + b"\0", np.uint8).copy()
    lens = np.array([len(b) for b in pk], np.int32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    Wseq = W.reshape(1, -1).astype(np.int32)
    coef_off, pcm_off, coef_len, pcm_len = lib.synthesis_layout(Wseq, bs, ch)
    carry = ctx.new_decode_carry(1)
    want = ctx.decode_packets_resume(Wseq, coef_off, coef_len, offs.reshape(1, -1), lens.reshape(1, -1), data,
                                     pcm_off, pcm_len, carry)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_tail, d_W = t(ctx.new_decode_carry(1)[0]), t(ctx.new_decode_carry(1)[1])
    d_pcm = torch.zeros((1, ch, pcm_len), dtype=torch.float32, device=dev)
    d_res = torch.zeros(coef_len, dtype=torch.float32, device=dev)
    keep = [t(Wseq), t(coef_off), t(offs), t(lens), t(data), t(pcm_off)]
    torch.cuda.synchronize()
    ctx.decode_packets_resume_dev(1, Wseq.shape[1], None, keep[0].data_ptr(), keep[1].data_ptr(), d_res.data_ptr(),
                                  keep[2].data_ptr(), keep[3].data_ptr(), keep[4].data_ptr(), keep[5].data_ptr(),
                                  d_pcm.data_ptr(), 0, pcm_len, d_tail.data_ptr(), d_W.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(d_pcm.cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert np.array_equal(d_tail.cpu().numpy().view(np.uint32), carry[0].view(np.uint32))
    assert np.array_equal(d_W.cpu().numpy(), carry[1])

    def bad(**kw):
        a = dict(Wseq=Wseq, coef_off=coef_off, res_len=coef_len, pkt_off=offs.reshape(1, -1),
                 pkt_bytes=lens.reshape(1, -1), data=data, pcm_off=pcm_off, pcm_stride=pcm_len,
                 carry=ctx.new_decode_carry(1))
        a.update(kw)
        with pytest.raises(lib.VB200Error, match="-131"):
            ctx.decode_packets_resume(**a)
    bad(pkt_bytes=(lens + np.int32(len(data))).reshape(1, -1))              # past the end of data
    bad(pkt_off=(offs - 1).reshape(1, -1))                                  # before it
    W2 = Wseq.copy()
    W2[0, 3] = 2
    bad(Wseq=W2)
    bad(res_len=coef_len - 1)
    k = ctx.new_decode_carry(1)
    k[1][:] = 3
    bad(carry=k)
    with pytest.raises(lib.VB200Error, match="-131"):
        ctx.decode_packets_resume(Wseq, coef_off, coef_len, offs.reshape(1, -1), lens.reshape(1, -1), data, pcm_off,
                                  pcm_len, ctx.new_decode_carry(1), count=np.array([Wseq.shape[1] + 1], np.int32))
    rc = ctx.L.vb200_decode_packets_resume(ctx.h, 1, Wseq.shape[1], None, Wseq.ctypes.data, coef_off.ctypes.data,
                                           coef_len, offs.ctypes.data, lens.ctypes.data, None, data.size,
                                           pcm_off.ctypes.data, want.ctypes.data, 0, pcm_len, None)
    assert rc == -131


def test_no_entropy_setup_is_an_error(cuda_ok):
    import os
    from conftest import ROOT
    from vorbis_b200 import abi
    setup = abi.SetupHolder.load(os.path.join(ROOT, "tests", "golden", "setup_44k_stereo_q5.npz"))
    ctx = lib.Context(setup, device=0)
    data = np.zeros(8, np.uint8)
    one = np.zeros((1, 1), np.int64)
    with pytest.raises(lib.VB200Error, match="entropy_setup"):
        ctx.decode_packets_resume(np.zeros((1, 1), np.int32), one, 4096, one, np.ones((1, 1), np.int32), data,
                                  one, 1, ctx.new_decode_carry(1))
    with pytest.raises(lib.VB200Error, match="entropy_setup"):
        ctx.decode_entropy(np.zeros(1, np.int32), one[0], np.ones(1, np.int32), data, one[0], 4096)


@pytest.mark.parametrize("ch,rate,q", DRIVER_CASES)
@pytest.mark.parametrize("s16", [False, True])
def test_driver_device_and_host_paths_equal_stock(cuda_ok, ch, rate, q, s16):
    _need()
    from test_gpu_decode_driver import _streams as driver_streams
    enc = driver_streams(ch, rate, q)
    want = [decode.stock_decode(p, audio, ch, s16=s16) for p, audio in enc]
    joined = decode.join([(p.buf, a, p.meta[:3]) for p, a in enc])
    rng = np.random.default_rng(ch * 1000 + int(q * 10))
    sched = rng.integers(0, 6, (400, len(enc)))
    for host in (False, True):
        got, st = dp.md_run(joined, sched, ch, s16=s16, host_entropy=host)
        assert st["entropy_on_device"] == (not host)
        assert st["max_launches_per_round"] <= 2
        for s in range(len(enc)):
            assert got[s].shape == want[s].shape
            assert np.array_equal(got[s].view(np.uint8), want[s].view(np.uint8)), "stream %d host=%s" % (s, host)


@pytest.mark.parametrize("ch,rate,q", DRIVER_CASES)
def test_driver_truncated_packets_mid_stream(cuda_ok, ch, rate, q):
    _need()
    p = decode.encode(ch, rate, q, probe_signal(ch, rate, 0.9, seed=77))
    audio = p.audio.copy()
    k = len(audio) // 2
    for j, frac in ((k - 3, 0.5), (k, 0.1), (k + 1, 0.0), (k + 4, 0.8)):
        audio[j, 1] = int(audio[j, 1] * frac)
    want = decode.stock_decode(p, audio, ch)
    joined = decode.join([(p.buf, audio, p.meta[:3])] * 3)
    got, st = dp.md_run(joined, np.full((30, 3), 2), ch)
    assert st["entropy_on_device"]
    for s in range(3):
        assert np.array_equal(got[s].view(np.uint32), want.view(np.uint32)), "stream %d" % s
