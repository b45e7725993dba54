"""Golden frames of user colour expressions from the REFERENCE ITSELF on Mesa llvmpipe (oracle/ref_gl.py): the reference's
own module shaders with the user's <module>.glsl (#define COLOR <expr>), compiled by Mesa's GLSL compiler, driven by the
reference's rd_update on synthetic PCM exactly as tests/golden/make_llvmpipe_golden.py does.  The expressions are those of
tests/color_programs.py that reach the domain edges (+-0, +-inf and NaN from 1 / (d - Z), log / log2 / sqrt / pow outside
their domain and on subnormals, sin / cos / tan of huge arguments, atan at the infinities, mod(x, 0), smoothstep(e, e, x),
comparisons with NaN), on bars 1280x720, graph 1280x720 and radial 1920x1080.

Writes tests/golden/color_expr_llvmpipe.npz:
  <case>_tex     [2][n] u16     what stage 1 samples for audio_l / audio_r after the last frame
  <case>_frame   [h][w][4] u8   the final frame (row 0 = bottom)
  <case>_params  JSON           the product's reading of the same configuration (glava_b200_load_config)
  <case>_cfg     JSON           {rc, files, seed, frames, ur}
  case_names, gl_strings

tests/test_color_programs.py replays the cases through the host build, tests/test_gpu_color_programs.py through the kernels.
Run in the build container only (needs /root/reference and the Nsight Compute Mesa):
    python tests/golden/make_color_expr_llvmpipe_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import ref_gl  # noqa: E402
from tests import color_programs as cp  # noqa: E402
import make_llvmpipe_golden as mk  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
EXPRS = ("inf_nan", "log_domain", "sqrt_pow", "trig_large", "atan_quadrants", "mod_smooth", "nan_cmp", "rounding")
SITES = (("bars", 1280, 720, "#define AMPLIFY 300\n"), ("graph", 1280, 720, "#define VSCALE 300\n"),
         ("radial", 1920, 1080, ""))


def cases():
    out = []
    for i, expr in enumerate(EXPRS):
        for j, (module, w, h, extra) in enumerate(SITES):
            text = extra + "#define COLOR " + cp.program_text(expr, module) + "\n"
            out.append((f"{module}_{expr}", mk.rc(module, 1024, w, h), {f"{module}.glsl": text}, 6, 300 + 10 * i + j))
    return out


KEEP = ("_tex", "_frame", "_params", "_cfg")


def main():
    assert ref_gl.available(), "needs oracle/_ref/libglava_ref_gl.so + the Nsight Compute Mesa"
    out, names = {}, []
    for name, rc_text, files, frames, seed in cases():
        rec = mk.run_case(name, rc_text, files, frames, seed)
        out.update({k: v for k, v in rec.items() if k.endswith(KEEP)})
        names.append(name)
    out["case_names"] = np.array(names)
    with ref_gl.ReferenceGL(rc=mk.rc("test", 256, 8, 8)) as r:
        out["gl_strings"] = np.array(list(r.gl_strings))
    path = os.path.join(HERE, "color_expr_llvmpipe.npz")
    np.savez_compressed(path, **out)
    print("wrote color_expr_llvmpipe.npz", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
