"""Writes tests/golden/ref/bitrate.npz: random packet-size sequences for every configuration of
oracle.bitrate.CONFIGS, the configuration's bitrate_manager_info and block sizes as the reference derives them, and
what the reference's own vorbis_bitrate_addblock / flushpacket make of them (choice, final bytes, state after every
block).  tests/test_bitrate_oracle.py checks the oracle against it where oracle/_ref was not built.

Run from the repository root after build(), where the reference sources exist:
    python tests/golden/make_golden_bitrate.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import __graft_entry__  # noqa: E402
from oracle import bitrate as B  # noqa: E402


def main():
    __graft_entry__.build()
    assert B.ref_available(), "oracle/_ref/libvorbis_ref_bitrate.so not built"
    rng = np.random.default_rng(31)
    out = {"names": np.array(list(B.CONFIGS))}
    info_int, info_float, bs_all, rates, configs = [], [], [], [], []
    for name, cf in B.CONFIGS.items():
        info, bs = B.ref_bitrate_info(cf)
        info_int.append([info.avg_rate, info.min_rate, info.max_rate, info.reservoir_bits])
        info_float.append([info.reservoir_bias, info.slew_damp])
        bs_all.append(bs)
        rates.append(cf.rate)
        configs.append(B.config_array(cf))
        lens, W, bits = B.size_sequences(rng, 60, bs, B.target_bits(info, bs, cf.rate))
        choice, nbytes, ok, after = B.ref_bitrate_replay(cf, lens, W, bits, seed=11)
        assert ok.all()
        out.update({name + "_lens": lens, name + "_W": W.astype(np.int8), name + "_bits": bits,
                    name + "_choice": choice.astype(np.int8), name + "_bytes": nbytes.astype(np.int32),
                    name + "_state": after.view(np.uint8).reshape(len(after), -1)})
    out.update({"info_int": np.array(info_int, np.int64), "info_float": np.array(info_float, np.float64),
                "bs": np.array(bs_all, np.int32), "rate": np.array(rates, np.int64),
                "config": np.array(configs, np.float64)})
    path = os.path.join(ROOT, "tests", "golden", "ref", "bitrate.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
