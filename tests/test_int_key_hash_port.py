"""The NumPy port of the integer keys' stored form and hash (tests/test_gpu_int_keys.py: int_key_hash), pinned against the device
header: a host program compiled with nvcc includes dnz_device.cuh and prints int_key's words and hash for a fixed value list.  The
GPU collision tests pick colliding integer keys with the port, so a port that drifted from the header would silently stop
producing collisions."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.test_gpu_int_keys import INT_KEY_TAG, int_key_hash

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "denormalized_b200", "csrc")


def _values():
    rng = np.random.default_rng(23)
    v = [0, 1, 2, 0xFFFFFFFF, 0x80000000, 0x7FFFFFFF, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, 424242]
    v += rng.integers(0, 1 << 63, 200, dtype=np.uint64).tolist() + rng.integers(0, 1 << 32, 100, dtype=np.uint64).tolist()
    return np.array(v, np.uint64)


def test_zero_keys_are_not_all_zero_words():
    # the tag keeps the stored key words of the value 0 away from the probe's torn-read marker (both words zero)
    assert INT_KEY_TAG != 0
    h4, h8 = int_key_hash(np.zeros(1, np.uint64), 4), int_key_hash(np.zeros(1, np.uint64), 8)
    assert h4[0] != h8[0]                                 # the width takes part in the hash


def test_int_key_port_matches_the_device_header(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    vals = _values()
    src = tmp_path / "int_key_probe.cu"
    src.write_text('#include <cstdio>\n#include "dnz_device.cuh"\n'
                   "static const unsigned long long V[] = {" + ",".join("%dull" % int(x) for x in vals) + "};\n"
                   "int main() {\n"
                   "  for (unsigned long long v : V)\n"
                   "    for (unsigned w : {4u, 8u}) {\n"
                   "      const dnz::KeyRef k = dnz::int_key(v, w);\n"
                   "      std::printf(\"%llu %llu %u %llu\\n\", (unsigned long long)k.k0, (unsigned long long)k.k1, k.len,\n"
                   "                  (unsigned long long)dnz::stored_key_hash(k.k0, k.k1, k.len) - k.hash);\n"
                   "      std::printf(\"%llu\\n\", (unsigned long long)k.hash);\n"
                   "    }\n  return 0;\n}\n")
    exe = tmp_path / "int_key_probe"
    subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src), "-o", str(exe)],
                   check=True, capture_output=True)
    lines = [ln for ln in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n") if ln.strip()]
    assert len(lines) == 4 * len(vals)
    for i, v in enumerate(vals):
        for j, w in enumerate((4, 8)):
            k0, k1, ln, d = (int(x) for x in lines[4 * i + 2 * j].split())
            h = int(lines[4 * i + 2 * j + 1])
            assert k0 == (int(v) & 0xFFFFFFFF if w == 4 else int(v)) and k1 == INT_KEY_TAG and ln == w
            assert d == 0                                 # the dictionary's stored-key hash of the stored form is int_key's hash
            assert h == int(int_key_hash(np.array([v], np.uint64), w)[0]), (int(v), w)
