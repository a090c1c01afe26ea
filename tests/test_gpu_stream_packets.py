"""The bitrate manager on the device (vb200_bitrate_addblocks[_dev]) against the CPU oracle, and whole streams to
packets (vb200_encode_streams_packets[_managed]) against stock encoders: every packet byte for byte with its
granulepos, e_o_s and packetno.  The stock-encoder comparisons need oracle/_ref (built where the reference sources
exist; the libraries travel)."""
import numpy as np
import pytest

from conftest import CONFIG_NAMES, REF_ARGS, ROOT, load_setup, probe_signal
from oracle import bitrate as B
from test_gpu_encode_packets import SETUPS, _driver
from test_gpu_encode_packets_managed import _dev_managed
from vorbis_b200 import abi, lib

pytestmark = pytest.mark.gpu

NB = abi.PACKETBLOBS
VB200_EINVAL = -131
FIXTURE = ROOT + "/tests/golden/ref/bitrate.npz"


def _fixture():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def _contexts():
    """name -> (Context, BitrateInfo) for every fixture configuration whose rate and block sizes a golden setup has"""
    f = _fixture()
    setups = {}
    for name in CONFIG_NAMES:
        s = load_setup(name)
        setups.setdefault((s.rate, s.blocksize(0), s.blocksize(1)), s)
    out = {}
    for i, name in enumerate(str(n) for n in f["names"]):
        key = (int(f["rate"][i]), int(f["bs"][i][0]), int(f["bs"][i][1]))
        if key in setups:
            ctx = lib.Context(setups[key])
            info = B.info_from_arrays(f["info_int"][i], f["info_float"][i])
            ctx.bitrate_setup(info)
            out[name] = (ctx, info)
    return out, f


def _pack(lens, W, bits, max_blocks):
    """sequences -> [ns][max_blocks] rows (count = lens)"""
    ns = len(lens)
    Wm = np.zeros((ns, max_blocks), np.int32)
    bm = np.zeros((ns, max_blocks, NB), np.int32)
    t = 0
    for i, n in enumerate(lens):
        Wm[i, :n], bm[i, :n] = W[t:t + n], bits[t:t + n]
        t += n
    return Wm, bm


def _oracle_rows(info, rate, bs, lens, W, bits, max_blocks):
    c = np.full((len(lens), max_blocks), -5, np.int32)
    b = np.full((len(lens), max_blocks), -5, np.int32)
    st = np.zeros(len(lens), abi.BITRATE_STATE_DTYPE)
    t = 0
    for i, n in enumerate(lens):
        if n:
            ci, bi, ai = B.vbo_bitrate_addblock(info, rate, bs, W[t:t + n], bits[t:t + n])
            c[i, :n], b[i, :n], st[i] = ci, bi, ai[-1]
        t += n
    return c, b, st


def test_chooser_equals_oracle(cuda_ok):
    """the fixture's sequences, one stream each, and 1000 random streams of different lengths (some empty): choice,
    final bytes and state equal the oracle's; entries past count are untouched; the _dev form equals the host form;
    one launch"""
    import torch
    ctxs, f = _contexts()
    assert {"abr", "cbr", "max", "cbr_small"} <= set(ctxs)
    rng = np.random.default_rng(9)
    try:
        for name, (ctx, info) in ctxs.items():
            i = [str(n) for n in f["names"]].index(name)
            bs, rate = [int(v) for v in f["bs"][i]], int(f["rate"][i])
            sets = [(f[name + "_lens"], f[name + "_W"].astype(np.int32), f[name + "_bits"])]
            lens, W, bits = B.size_sequences(rng, 1000, bs, B.target_bits(info, bs, rate), max_len=40)
            lens[rng.random(1000) < 0.1] = 0
            W, bits = W[:lens.sum()], bits[:lens.sum()]
            sets.append((lens, W, bits))
            for lens, W, bits in sets:
                mb = int(lens.max()) + 3
                Wm, bm = _pack(lens, W, bits, mb)
                want_c, want_b, want_s = _oracle_rows(info, rate, bs, lens, W, bits, mb)
                st = ctx.bitrate_init(len(lens))
                c = np.full((len(lens), mb), -5, np.int32)
                b = np.full((len(lens), mb), -5, np.int32)
                l0 = ctx.launch_count()
                ctx.bitrate_addblocks(lens, Wm, bm, st, c, b)
                assert ctx.launch_count() - l0 == 1
                assert np.array_equal(c, want_c), name + ": choice"
                assert np.array_equal(b, want_b), name + ": bytes"
                nz = lens > 0
                for fld in ("avg_reservoir", "minmax_reservoir", "avgfloat", "choice"):
                    assert np.array_equal(st[fld][nz], want_s[fld][nz]), name + ": state " + fld
                fresh = ctx.bitrate_init(1)
                assert (st[~nz] == fresh[0]).all()
                # the _dev form
                d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
                     (("n", lens.astype(np.int32)), ("W", Wm), ("b", bm), ("s", ctx.bitrate_init(len(lens)).view(np.uint8)),
                      ("c", np.full_like(c, -5)), ("y", np.full_like(b, -5)))}
                ctx.bitrate_addblocks_dev(len(lens), mb, d["n"].data_ptr(), d["W"].data_ptr(), d["b"].data_ptr(),
                                          d["s"].data_ptr(), d["c"].data_ptr(), d["y"].data_ptr())
                torch.cuda.synchronize()
                assert np.array_equal(d["c"].cpu().numpy(), c) and np.array_equal(d["y"].cpu().numpy(), b)
                assert np.array_equal(d["s"].cpu().numpy().view(abi.BITRATE_STATE_DTYPE), st)
    finally:
        for ctx, _ in ctxs.values():
            ctx.close()


def test_chooser_cut_into_calls_equals_one_call(cuda_ok):
    """every stream's blocks cut into 2-5 calls (different cuts per stream) that carry the state: one call's result"""
    ctxs, f = _contexts()
    rng = np.random.default_rng(12)
    try:
        for name, (ctx, info) in ctxs.items():
            i = [str(n) for n in f["names"]].index(name)
            bs, rate = [int(v) for v in f["bs"][i]], int(f["rate"][i])
            lens, W, bits = B.size_sequences(rng, 200, bs, B.target_bits(info, bs, rate), max_len=60)
            mb = int(lens.max())
            Wm, bm = _pack(lens, W, bits, mb)
            st1 = ctx.bitrate_init(len(lens))
            c1, b1 = ctx.bitrate_addblocks(lens, Wm, bm, st1)
            st = ctx.bitrate_init(len(lens))
            c = np.zeros_like(c1)
            b = np.zeros_like(b1)
            cuts = [np.sort(np.r_[0, rng.integers(0, n + 1, rng.integers(1, 5)), n]) for n in lens]
            for piece in range(5):
                cnt = np.array([cu[piece + 1] - cu[piece] if piece + 1 < len(cu) else 0 for cu in cuts], np.int32)
                start = np.array([cu[piece] if piece + 1 < len(cu) else 0 for cu in cuts])
                Wp = np.zeros_like(Wm)
                bp = np.zeros_like(bm)
                for s in range(len(lens)):
                    Wp[s, :cnt[s]] = Wm[s, start[s]:start[s] + cnt[s]]
                    bp[s, :cnt[s]] = bm[s, start[s]:start[s] + cnt[s]]
                cp, yp = ctx.bitrate_addblocks(cnt, Wp, bp, st)
                for s in range(len(lens)):
                    c[s, start[s]:start[s] + cnt[s]] = cp[s, :cnt[s]]
                    b[s, start[s]:start[s] + cnt[s]] = yp[s, :cnt[s]]
            assert np.array_equal(c, c1) and np.array_equal(b, b1), name
            assert (st == st1).all(), name
    finally:
        for ctx, _ in ctxs.values():
            ctx.close()


def _timelines(caps, ch):
    stride = (max(c["timeline"].shape[1] for c in caps) + 3) & ~3
    tl = np.zeros((len(caps), ch, stride), np.float32)
    for i, c in enumerate(caps):
        tl[i, :, :c["timeline"].shape[1]] = c["timeline"]
    pcm_len = np.array([c["timeline"].shape[1] for c in caps], np.int64)
    eof = np.array([c["eof"] for c in caps], np.int64)
    return tl, pcm_len, eof


def _compare(got, caps, what, eos=True):
    for i, c in enumerate(caps):
        n = int(got["nblocks"][i])
        info = got["info"][i, :n]
        assert n == len(c["packets"]) if eos else n <= len(c["packets"]), "%s stream %d: %d blocks" % (what, i, n)
        assert got["packets"][i] == c["packets"][:n], "%s stream %d: packet bytes" % (what, i)
        assert np.array_equal(info["packetno"], c["packetno"][:n]), "%s stream %d: packetno" % (what, i)
        if eos:
            assert np.array_equal(info["granulepos"], c["granulepos"]), "%s stream %d: granulepos" % (what, i)
            assert np.array_equal(info["e_o_s"], c["e_o_s"]), "%s stream %d: e_o_s" % (what, i)
        else:
            assert not info["e_o_s"].any()
            keep = c["e_o_s"][:n] == 0
            assert np.array_equal(info["granulepos"][keep], c["granulepos"][:n][keep]), "%s stream %d" % (what, i)


def _need_ref():
    if not B.ref_available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")


def _streams(ch, rate, secs):
    from test_plan_vs_ref import burst_signal
    n = int(rate * secs)
    return [probe_signal(ch, rate, secs, seed=3)[:, :n], burst_signal(ch, rate, secs, 5)[:, :n],
            np.random.default_rng(4).uniform(-0.5, 0.5, (ch, rate // 50)).astype(np.float32),   # shorter than a long block
            np.zeros((ch, n // 2), np.float32)]                            # silence


@pytest.mark.parametrize("ch,rate,q", SETUPS)
def test_unmanaged_whole_streams(cuda_ok, ch, rate, q):
    """vb200_encode_streams_packets on the stock VBR encoder's timelines: the stock encoder's packets, granulepos,
    e_o_s and packetno, stream by stream; without EOF, its first nblocks packets with e_o_s 0; a bounded number of
    launches"""
    _need_ref()
    d = _driver(ch, rate, q)
    ctx = d.ctx
    try:
        caps = [B.ref_stream_capture(B.vbr(ch, rate, q), p) for p in _streams(ch, rate, 0.6)]
        tl, pcm_len, eof = _timelines(caps, ch)
        l0 = ctx.launch_count()
        got = ctx.encode_streams_packets(tl, pcm_len, eof)
        launches = ctx.launch_count() - l0
        _compare(got, caps, "q=%g" % q)
        assert (got["info"]["choice"][got["info"]["bytes"] > 0] == NB // 2).all()
        # the same streams cut at their EOF sample and passed without EOF
        noeof = ctx.encode_streams_packets(tl, np.minimum(pcm_len, eof), None)
        _compare(noeof, caps, "no EOF", eos=False)
        # launches do not grow with the stream count
        more = ctx.encode_streams_packets(np.concatenate([tl] * 3), np.concatenate([pcm_len] * 3),
                                          np.concatenate([eof] * 3))
        assert more["packets"] == got["packets"] * 3
        l1 = ctx.launch_count()
        ctx.encode_streams_packets(np.concatenate([tl] * 3), np.concatenate([pcm_len] * 3), np.concatenate([eof] * 3))
        assert ctx.launch_count() - l1 == launches <= 40
    finally:
        d.close()


def _noise_and_silence(ch, rate, secs, seed):
    rng = np.random.default_rng(seed)
    n = int(rate * secs)
    pcm = rng.uniform(-0.9, 0.9, (ch, n)).astype(np.float32)
    seg = rate // 4
    for a in range(seg, n, 2 * seg):
        pcm[:, a:a + seg] = 0
    return pcm


MANAGED = [
    ("abr", 2, 44100, -1, 128000, -1, None),
    ("mono64", 1, 44100, -1, 64000, -1, None),
    ("cbr", 2, 44100, 128000, 128000, 128000, None),
    ("cbr_small", 2, 44100, 128000, 128000, 128000, (4000, 0.3, 0.5)),
]


@pytest.mark.parametrize("name,ch,rate,max_br,nominal,min_br,rm2", MANAGED)
def test_managed_whole_streams(cuda_ok, name, ch, rate, max_br, nominal, min_br, rm2):
    """vb200_encode_streams_packets_managed on a stock managed encoder's timelines: its packets, granulepos, e_o_s and
    packetno, stream by stream.  With a small reservoir on loud noise and silence, at least one kept packet is cut short
    and one padded (against the kept curve's natural length)"""
    _need_ref()
    if not B.ref_available(True):
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    cf = B.managed(ch, rate, max_br, nominal, min_br, *(rm2 or ()))
    info, _ = B.ref_bitrate_info(cf)
    d = B.ManagedDriver(ch, rate, max_br, nominal, min_br)
    ctx = d.ctx
    try:
        ctx.bitrate_setup(info)
        sig = _streams(ch, rate, 0.8)
        if rm2:
            sig = [_noise_and_silence(ch, rate, 1.5, 1), _noise_and_silence(ch, rate, 1.0, 2)] + sig
        caps = [B.ref_stream_capture(cf, p) for p in sig]
        tl, pcm_len, eof = _timelines(caps, ch)
        got = ctx.encode_streams_packets(tl, pcm_len, eof, managed=True)
        _compare(got, caps, name)
        if rm2:
            # natural lengths of the kept curves: the streams chain and the managed coder on their own
            ch_out = ctx.encode_streams_managed(tl, pcm_len, eof)
            nat = {}
            for W in (0, 1):
                cnt = ch_out["count"][W]
                if not cnt:
                    continue
                desc = np.zeros(cnt, abi.BLOCKDESC_DTYPE)
                plan = ch_out["plan"]
                for s in range(len(caps)):
                    for b in plan[s, :ch_out["nblocks"][s]]:
                        if b["W"] == W:
                            desc["lW"][b["slot"]], desc["nW"][b["slot"]] = b["lW"], b["nW"]
                g = ch_out[W]
                rc, _, bits = _dev_managed(ctx, W, desc, g["posts"], g["nonzero"], g["iwork"])
                assert rc == 0
                nat[W] = (bits + 7) // 8
            cut = pad = 0
            for s in range(len(caps)):
                for k in range(got["nblocks"][s]):
                    b, r = got["plan"][s, k], got["info"][s, k]
                    natural = nat[int(b["W"])][r["choice"], b["slot"]]
                    cut += r["bytes"] < natural
                    pad += r["bytes"] > natural
            print("%s: %d truncated, %d padded packets" % (name, cut, pad))
            assert cut > 0 and pad > 0
    finally:
        d.close()


def test_errors(cuda_ok):
    """VB200_EINVAL without an entropy setup, without a bitrate setup (managed), for an un-managed bitrate setup, for a
    small data_cap (info filled), for outputs that are not NULL and for null pointers"""
    ctx = lib.Context(load_setup("44k_stereo_q5"))
    try:
        ch, rate, q = REF_ARGS["44k_stereo_q5"]
        pcm = probe_signal(ch, rate, 0.3, seed=1)
        tl = np.zeros((1, ch, pcm.shape[1] + 4096), np.float32)
        tl[0, :, 1024:1024 + pcm.shape[1]] = pcm
        pcm_len = np.array([tl.shape[2]], np.int64)
        L = ctx.L
        assert ctx.encode_streams_packets(tl, pcm_len, data_cap=1 << 20, check=False)["rc"] == VB200_EINVAL
        assert L.vb200_bitrate_init(ctx.h, np.zeros(1, abi.BITRATE_STATE_DTYPE).ctypes.data) == VB200_EINVAL
        assert L.vb200_bitrate_addblocks(ctx.h, 1, 1, None, None, None, None, None, None) == VB200_EINVAL
        unmanaged = abi.BitrateInfo(128000, -1, -1, 0, 0.1, 1.5)
        ctx.bitrate_setup(unmanaged)
        assert L.vb200_bitrate_init(ctx.h, np.zeros(1, abi.BITRATE_STATE_DTYPE).ctypes.data) == VB200_EINVAL
        assert L.vb200_bitrate_setup(ctx.h, None) == VB200_EINVAL
        assert L.vb200_bitrate_init(None, None) == VB200_EINVAL
        assert L.vb200_encode_streams_packets(ctx.h, 1, 7, None, None, None, 0) == VB200_EINVAL
        assert L.vb200_encode_streams_packets_managed(ctx.h, 1, None, None, None, 0) == VB200_EINVAL
    finally:
        ctx.close()
    _need_ref()
    d = _driver(2, 44100, 0.5)
    ctx = d.ctx
    try:
        cap = B.ref_stream_capture(B.vbr(2, 44100, 0.5), probe_signal(2, 44100, 0.5, seed=2))
        tl, pcm_len, eof = _timelines([cap], 2)
        full = ctx.encode_streams_packets(tl, pcm_len, eof)
        small = ctx.encode_streams_packets(tl, pcm_len, eof, data_cap=100, check=False)
        assert small["rc"] == VB200_EINVAL
        assert np.array_equal(small["info"], full["info"])
        # managed without a bitrate setup, then with an un-managed one
        assert ctx.encode_streams_packets(tl, pcm_len, eof, managed=True, check=False)["rc"] == VB200_EINVAL
        ctx.bitrate_setup(abi.BitrateInfo(128000, -1, -1, 0, 0.1, 1.5))
        assert ctx.encode_streams_packets(tl, pcm_len, eof, managed=True, check=False)["rc"] == VB200_EINVAL
        st = np.zeros(1, abi.BITRATE_STATE_DTYPE)
        assert ctx.bitrate_addblocks([1], np.zeros((1, 1)), np.zeros((1, 1, NB)), st, check=False) == VB200_EINVAL
        # posts given: the outputs stay in device scratch
        io = abi.StreamsIO()
        io.posts[0] = tl.ctypes.data
        info = np.zeros(8, abi.PACKET_INFO_DTYPE)
        assert ctx.L.vb200_encode_streams_packets(ctx.h, 1, 7, io, info.ctypes.data, None, 0) == VB200_EINVAL
    finally:
        d.close()
