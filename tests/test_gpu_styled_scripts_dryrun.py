"""CPU tier: the styled raster -m gpu script (tests/test_gpu_styled_raster_variants.py: every launch variant under stream
styles, the coverage assertions, the styled dirty-row sequences) run against the emulation-backed Renderer of
tools/dryrun_gpu_tests.py, whose streams render at their styled parameters, so that the style plumbing and coverage claims
of that script are checked without a device."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_styled_raster_script_passes_against_the_emulation_backed_renderer(built):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dryrun_gpu_tests.py"),
                          "tests/test_gpu_styled_raster_variants.py"], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert " passed" in out.stdout and "failed" not in out.stdout
