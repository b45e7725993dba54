"""Development aid: run the raster_textures-based -m gpu tests against a fake Renderer built on the host emulation (tests/emul),
to validate the test scripts themselves (golden keys, expectations, parameter plumbing) when no GPU is at hand.  The device
plumbing stays untested, of course.

    python tools/dryrun_gpu_tests.py                  # the scripts of SCRIPTS
    python tools/dryrun_gpu_tests.py tests/x.py ...    # these scripts instead (paths relative to the repository root)
"""
import sys, ctypes as C
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, pytest
import glava_b200 as g
from tests import emul

_frames = {}      # the fake ignores the environment: a launch-variant test rasters the same inputs once per variant


class Fake:
    def __init__(self, params, batch=1, device=0):
        rc = g.lib().glava_b200_load_config  # noqa
        self.params = params.copy(); self.batch = batch; self.nsz = params.n; self._launch = 0; self._h = 1
        self.frames = [None] * batch
        self.styles = [g.StreamStyle() for _ in range(batch)]
    # stream styles: stream s renders what a renderer of style_params(params, style_s) renders
    def set_stream_styles(self, streams, styles):
        streams, styles = list(streams), list(styles)
        assert len(streams) == len(styles) and len(set(streams)) == len(streams)
        for s, st in zip(streams, styles):
            assert 0 <= s < self.batch
            g.style_params(self.params, st)                       # refused styles raise, as the library's call does
            self.styles[s] = g.stream_style(st)
    def get_stream_styles(self, streams):
        return [self.styles[s] for s in streams]
    def _stream_params(self, s):
        return g.style_params(self.params, self.styles[s]) if self.styles[s].set else self.params
    def raster_textures(self, tl, tr=None):
        tl = np.asarray(tl); tr = tl if tr is None else np.asarray(tr)
        for s in range(self.batch):
            q = self._stream_params(s)
            key = (bytes(q), tl[s].tobytes(), tr[s].tobytes())
            if key not in _frames:
                _frames[key] = emul.raster(q, tl[s], tr[s])
            self.frames[s] = _frames[key].copy()
        self._launch += self._raster_launches()
    def _raster_launches(self):
        """the launches the library plans for this raster pass (raster_plan.h, through the host build); a host build that
        does not export the plan counts one launch per pass, which is all the test scripts written against it check"""
        if not hasattr(emul, "raster_plan"):
            return 1
        env = {k[len("GLAVA_B200_"):]: v for k, v in os.environ.items() if k.startswith("GLAVA_B200_")}
        slots = self.params.fb_slots if 0 < self.params.fb_slots < self.batch else self.batch
        return emul.raster_plan(self.params, self.batch, slots, env)["launches"]
    def readback(self, s=0, out=None): return self.frames[s]
    # update() / textures(): the oracle's whole-rd_update restatement stands in for the spectrum kernels (script logic only)
    def update(self, lb, rb=None, modified=True):
        from oracle.oracle import Oracle, OracleStream, ext_from, params_from
        if not hasattr(self, "_streams"):
            o = Oracle("pm")
            self._streams = [OracleStream(o, params_from(self.params), ext_from(self.params)) for _ in range(self.batch)]
        rb = lb if rb is None else rb
        self._tex = [st.update(lb[s], rb[s], modified)[2:] for s, st in enumerate(self._streams)]
        self.nsz = self._streams[0].n
        self.frames = [emul.raster(self._stream_params(s), t[0], t[1]) for s, t in enumerate(self._tex)]
    def textures(self):
        return np.stack([t[0] for t in self._tex]), np.stack([t[1] for t in self._tex])
    def reconfigure(self, p): self.params = p.copy(); self._launch += 1
    @property
    def launch_count(self): return self._launch
    def close(self): pass
    def __enter__(self): return self
    def __exit__(self, *a): pass

g.Renderer = Fake
import glava_b200.api as api
api.Renderer = Fake
# Pipe.apply goes through the C ABI with a real handle: emulate with params re-evaluation
def fake_apply(self, renderer):
    if getattr(self, "_last", None) == self.binds():
        return
    self._last = self.binds(); renderer.reconfigure(self.params())
api.Pipe.apply = fake_apply
SCRIPTS = ["tests/test_zz_gpu_blend.py", "tests/test_zz_gpu_color_expr.py", "tests/test_zz_gpu_pipe.py", "tests/test_glsl_golden.py",
           "tests/test_zz_rd_golden.py", "tests/test_llvmpipe_golden.py", "tests/test_gpu_raster_variants.py"]
sys.exit(pytest.main(["-x", "-q", "-m", "gpu", "-p", "no:cacheprovider"] +
                     [os.path.join(ROOT, f) for f in (sys.argv[1:] or SCRIPTS)]))
