"""bench.py's reference arm (`--impl reference`: the oracle port of the reference's CPU path, the one leg of the bench that runs without a
GPU) prints ONE JSON line with the contract's keys; and the GPU arm's roofline inputs are what it documents."""

import json
import os
import subprocess
import sys

import pytest

from conftest import ROOT


@pytest.mark.timeout(600)
def test_reference_arm_prints_one_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '0'],
                       capture_output=True, text=True, timeout=560, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('{')]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['unit'] == 'frames/s' and d['higher_is_better'] is True and d['value'] > 0
    assert d['metric'].startswith('rendered frames/sec') and d['steps'] == 1 and d['gpu_launches'] == 0
    assert d['cpu_baseline']['kind'] == 'port' and d['cpu_baseline']['cores'] >= 1 and d['cpu_baseline']['value'] == d['value']
    assert d['e2e'] == {'value': d['value'], 'unit': 'frames/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}


def test_roofline_inputs():
    """Algorithmic bytes per frame: both tri-planes once + the 53 output floats per ray.  No measured DRAM-traffic capture of the
    current ray-march kernel is committed, and the bench must say so instead of citing one."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('bench_mod', os.path.join(ROOT, 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    traffic, src = bench.raymarch_traffic()
    assert (traffic is None) == (not os.path.exists(bench.TRAFFIC_JSON)) and isinstance(src, str)
    assert bench.FRAME_ALGO_BYTES == 2 * 96 * 256 * 256 * 4 + 64 * 64 * 53 * 4
