"""CPU-side checks of round-2 host logic: the collective roofline arithmetic of bench.py and the NVLink measurement's
degenerate case."""
import importlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_collective_roofline_uses_the_measured_link():
    sys.path.insert(0, ROOT)
    bench = importlib.import_module("bench")
    wire = 22_384_640
    r = bench._roofline(150.0, wire, 8, 673.0)
    assert "measured in this run" in r["bound"]
    floor = (7 / 8) * wire / 673e9 * 1e6
    assert abs(r["floor_us"] - floor) < 1e-6 and abs(r["fraction_of_measured"] - floor / 150.0) < 1e-9
    r = bench._roofline(150.0, wire, 8)                 # no measurement: the H100 SXM data sheet's 450 GB/s per direction
    assert "450" in r["bound"] and abs(r["floor_us"] - (7 / 8) * wire / 450e9 * 1e6) < 1e-6
    r1 = bench._roofline(85.0, wire, 1)                  # one GPU: the bound is local HBM
    assert r1["bound"] == "hbm" and 0 < r1["fraction_of_measured"] < 1
    assert bench._roofline(0.0, wire, 8) is None


def test_link_measurement_needs_peers():
    from baton_b200.parallel.symm import SymmetricBuffer
    buf = SymmetricBuffer(1 << 12, "cpu")
    assert buf.world == 1 and buf.measure_link_gbps() is None and not buf.has_multicast
