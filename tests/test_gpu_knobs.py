"""Every tuning knob of DESIGN 6b at a non-default setting (-m gpu).  The library reads its knobs once per process, so each
setting runs tests/knob_child.py in a child process of its own; the child exits by itself, non-zero on any mismatch with
the compiled reference."""
import os
import subprocess
import sys

import pytest
import torch

from gpu_common import checker

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _max_rows_a():
    """the largest pass-A row budget the device's per-block shared-memory opt-in limit holds (with the 8 KB output staging)"""
    optin = getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", 232448)
    return (optin - (8 * 256 * 4 + 1280 + 8 * 32 * 32)) // 128


SETTINGS = [
    {"FSEB200_HUFD_ROWS": "160", "FSEB200_HUFD_ROWS_B": "0"},          # single pass: every table above 160 rows is hard
    {"FSEB200_HUFD_ROWS": "160"},                                       # heavy pass B
    {"FSEB200_HUFD_ROWS_B": "0"},
    {"FSEB200_HUFD_ROWS": "max"},
    {"FSEB200_HUFD_ROWS": "1700"},                                      # above the device maximum: clamped
    {"FSEB200_ENC_EK": "8"},
    {"FSEB200_HOST_CHUNK_BLOCKS": "64"},
]


@pytest.mark.parametrize("setting", SETTINGS, ids=lambda s: ",".join("%s=%s" % (k[8:], v) for k, v in s.items()))
def test_knob_setting(setting):
    if not checker()[1]:
        pytest.skip("compares against the compiled reference")
    env = {k: v for k, v in os.environ.items() if not k.startswith("FSEB200_")}
    env.update({k: (str(_max_rows_a()) if v == "max" else v) for k, v in setting.items()})
    p = subprocess.run([sys.executable, os.path.join(HERE, "knob_child.py")], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (setting, p.stdout[-2000:], p.stderr[-4000:])
    assert "knob sweep ok" in p.stdout
