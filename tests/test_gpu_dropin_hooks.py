"""GPU: the UNMODIFIED reference façade (HectorSlamProcessor::update) with recording draw / debug hooks, on the
reference's CPU maps and with MapRepB200 plugged in — the hook call sequences must agree (oracle/dropin_hooks_check.cpp,
compiled from the reference headers in the build container, run here as a prebuilt binary)."""
import os
import subprocess

import pytest

from conftest import ROOT, report

pytestmark = pytest.mark.gpu
BIN = os.path.join(ROOT, "oracle", "_ref", "dropin_hooks_check")


def test_reference_facade_hooks_with_b200_maprep(hsb_lib):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/dropin_hooks_check not built (needs the reference headers at build time)")
    out = subprocess.run([BIN, "60"], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    for line in out.stdout.splitlines():
        report("dropin_hooks_check: " + line.strip())
    assert out.returncode == 0 and "HOOKS OK" in out.stdout, out.stdout + out.stderr
