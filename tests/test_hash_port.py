"""The NumPy port of the dictionary hash (tests/helpers.py: hash_words / hash_inline), pinned against the device header: a
host program compiled with nvcc includes dnz_device.cuh and prints the hashes of a fixed key list.  The GPU collision tests pick
colliding keys with the port, so a port that drifted from the header would silently stop producing collisions."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.helpers import hash_inline, hash_keys, key_words

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "denormalized_b200", "csrc")


def _nvcc():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return p if os.path.exists(p) else None


def _keys():
    rng = np.random.default_rng(11)
    keys = [b"", b"\0", b"\0" * 16, b"a", b"a\0", b"a\0\0", b"\0a", b"sensor_0", b"sensor_1234567", b"sensor_12345678",
            b"x" * 15 + b"\xff", b"\xff" * 16, b"0123456789abcdef"]
    keys += [bytes(rng.integers(0, 256, int(rng.integers(0, 17)), dtype=np.uint8)) for _ in range(200)]
    return keys


def test_hash_port_known_values():
    # equal-looking keys must hash apart through the length; zero padding makes "a" and "a\0" share their words
    h = hash_keys([b"a", b"a\0", b"a\0\0", b""] + [b"\0" * n for n in range(1, 17)])
    assert len(set(h.tolist())) == len(h)
    w = key_words([b"a", b"a\0"])
    assert np.array_equal(w[0], w[1])


def test_hash_port_matches_the_device_header(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    keys = _keys()
    w = key_words(keys)
    rows = ",\n".join("{%du,%du,%du,%du,%du}" % (w[i, 0], w[i, 1], w[i, 2], w[i, 3], len(k)) for i, k in enumerate(keys))
    src = tmp_path / "hash_probe.cu"
    src.write_text('#include <cstdio>\n#include "dnz_device.cuh"\n'
                   "static const unsigned K[][5] = {\n" + rows + "\n};\n"
                   "int main() {\n"
                   "  for (const auto& k : K) {\n"
                   "    const unsigned long long k0 = k[0] | ((unsigned long long)k[1] << 32), k1 = k[2] | ((unsigned long long)k[3] << 32);\n"
                   "    std::printf(\"%u %llu\\n\", dnz::hash_words(k[0], k[1], k[2], k[3], k[4]), (unsigned long long)dnz::hash_inline(k0, k1, k[4]));\n"
                   "  }\n  return 0;\n}\n")
    exe = tmp_path / "hash_probe"
    subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src), "-o", str(exe)],
                   check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    dev = np.array([[int(x) for x in line.split()] for line in out if line.strip()], np.uint64)
    assert dev.shape == (len(keys), 2)
    port = hash_keys(keys)
    k0 = w[:, 0].astype(np.uint64) | (w[:, 1].astype(np.uint64) << np.uint64(32))
    k1 = w[:, 2].astype(np.uint64) | (w[:, 3].astype(np.uint64) << np.uint64(32))
    assert np.array_equal(dev[:, 0], port.astype(np.uint64))
    assert np.array_equal(dev[:, 1], hash_inline(k0, k1, np.array([len(k) for k in keys], np.uint32)).astype(np.uint64))
