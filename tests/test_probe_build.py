"""CPU: the probe library (tests/device/hsb_probe.cu, the scalar device functions for test_gpu_scalar_functions.py) is
compiled with exactly the product library's nvcc flags — -fmad=false above all — so a probed function is generated as
the kernels generate it, and the two builds cannot drift apart.  Nothing in the package loads the probe."""
import os

from conftest import ROOT


def test_probe_uses_product_flags():
    from hector_slam_b200 import build

    cmd = build.probe_command()
    flags = build.NVCC_FLAGS
    assert os.path.basename(cmd[0]) == "nvcc"
    assert cmd[1:1 + len(flags)] == flags, cmd
    rest = cmd[1 + len(flags):]
    assert rest == ["-I", build.CSRC, "-o", build.PROBE_LIB, build.PROBE_SRC], rest
    assert "-fmad=false" in flags and "arch=compute_90a,code=sm_90a" in flags
    assert os.path.dirname(build.PROBE_LIB) == os.path.dirname(build.LIB)


def test_package_never_loads_the_probe():
    pkg = os.path.join(ROOT, "hector_slam_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")) and f != "build.py":
                text = open(os.path.join(d, f), encoding="utf-8").read()
                assert "hsb200_probe" not in text and "PROBE_LIB" not in text and "hsb_probe_" not in text, f
