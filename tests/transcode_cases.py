"""Shared by tests/test_jpeg_transcode_host.py and tests/test_gpu_jpeg_transcode.py: the CPU build of
the transcode bodies (tests/harness/host_jpeg_transcode.cu), a runner for it and the restart
intervals both sweep."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from tests.conftest import ROOT

OK, UNSUPPORTED, MALFORMED = 0, 1, 2
INTERVALS = [1, 3, 17, 0, 65535]          # 0: auto; 65535 is at least every fixture's MCU count
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17"]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    return nvcc


def _build(tmp_path_factory, name, extra):
    exe = str(tmp_path_factory.mktemp("harness") / name)
    r = subprocess.run([_nvcc()] + FLAGS + extra + ["-o", exe,
                        os.path.join(ROOT, "tests", "harness", "host_jpeg_transcode.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _runner(exe):
    def run(blobs, R, env=None):
        inp = struct.pack("<i", len(blobs)) + b"".join(struct.pack("<q", len(b)) + bytes(b) for b in blobs)
        out = subprocess.run([exe, str(R)], input=inp, capture_output=True, env=env)
        assert out.returncode == 0, out.stderr
        res, pos = [], 0
        for _ in blobs:
            st, ri, nint, eq, out_ri, out_nseg = struct.unpack_from("<6i", out.stdout, pos)
            size, = struct.unpack_from("<q", out.stdout, pos + 24)
            pos += 32
            data = out.stdout[pos:pos + size]
            pos += size
            n = nint if st == OK else 0
            bits = np.frombuffer(out.stdout, np.int32, n, pos)
            pos += 4 * n
            res.append(dict(status=st, ri=ri, nint=nint, coef_equal=eq, out_ri=out_ri, out_nseg=out_nseg, out=data,
                            bits=bits))
        assert pos == len(out.stdout)
        return res
    return run
