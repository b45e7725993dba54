"""Shared case list for the colour-expression programs (DESIGN §4.5): user COLOR / BAR_OUTLINE macros compiled into
glava_b200_color_prog and run by raster_core.h eval_color_prog in the bars / graph row tables, the radial geometry cache,
the generic and radial per-pixel kernels, their non-native-opacity forms and their styled twins.

PROGRAMS are hand-written expressions over `d` that reach the edges of each operation: +-0, +-inf and NaN from
1 / (d - Z) and 0 * that (Z is a d the module's rows hit exactly), exp overflow and exp(-d) falling through the subnormals,
log / log2 / sqrt / pow of negative, zero, subnormal and infinite values, sin / cos / tan far past 2^31 pi/2, atan in all four
quadrants and at the infinities, mod(x, 0), smoothstep(e, e, x), NaN through min / max / clamp / step, the comparisons and
the selects, and programs at the 8-register and 64-instruction limits.  EdgeGen adds seeded random ones.  CASES put them
at sites (module, size, options, environment, styles); tests/test_color_programs.py computes from the compiled programs and
from the raster plan that together they reach every opcode and every kernel form, and tests/test_gpu_color_programs.py runs
them on the device."""
import os
import tempfile

import numpy as np

import glava_b200 as g
from tests.test_color_expr import _Gen

N = 1024
OPS = ("SPLAT", "VAR", "LANE", "SHUF", "ADD", "SUB", "MUL", "DIV", "MIN", "MAX", "MOD", "STEP", "NEG", "ABS", "FLOOR", "CEIL",
       "FRACT", "SQRT", "SIN", "COS", "LOG", "SIGN", "TRUNC", "MIX", "CLAMP", "SMOOTHSTEP", "LT", "LE", "EQ", "NE", "AND", "OR",
       "NOT", "SELECT", "EXP", "EXP2", "LOG2", "POW", "ATAN2", "TAN")        # include/glava_b200.h GLAVA_B200_COP_*
assert len(OPS) == 40

# {z}: a value of d on one row of the module (bars: row centres t + 0.5; graph: integer rows; radial: not hit exactly)
PROGRAMS = {
    "inf_nan": "vec4(1.0 / (d - {z}), 0.0 * (1.0 / (d - {z})) + 0.5, step(0.0, -1.0 / (d - {z})), sign(-0.0 * d) + 0.75)",
    "exp_range": "vec4(exp(d) * 1e-38, exp(-d) * 1e38, exp2(d - 130.0), exp(-d * 0.5) * 1e20)",
    "log_domain": "vec4(log(d - {z}) * 0.2, log2(d - {z}) * 0.05 + 0.5, log(exp(-d)) * -0.01, log(exp(d)) * 0.005)",
    "sqrt_pow": "vec4(sqrt(d - {z}) * 0.1, pow(d - {z}, 0.5) * 0.1, pow(exp(d), -0.01), pow(0.0 * d, 2.0) + pow(d * 1e-20, 2.0) * 1e36)",
    "trig_large": "vec4(sin(d * 1e3) * 0.5 + 0.5, cos(d * 1e6) * 0.5 + 0.5, tan(d * 1e9) * 0.05 + 0.5, sin(d * 1e6) * 0.5 + 0.5)",
    "atan_quadrants": "vec4(atan(sin(d * 0.05), cos(d * 0.05)) * 0.15 + 0.5, atan(1.0 / (d - {z}), -1.0 / (d - {z})) * 0.15 + 0.5, "
                      "atan(exp(d), -exp(d)) * 0.15 + atan(d - {z}) * 0.1 + 0.5, atan(-exp(d), exp(d * 0.5)) * 0.15 + 0.5)",
    "mod_smooth": "vec4(mod(d, 0.0), smoothstep(20.5, 20.5, d), smoothstep(30.0, 10.0, d), mod(-d, 7.0) / 7.0)",
    "nan_ops": "vec4(min(sqrt({z} - d), 0.5), max(sqrt({z} - d), 0.5), clamp(sqrt({z} - d), 0.25, 0.75), step(sqrt({z} - d), 2.0))",
    "nan_cmp": "vec4(sqrt({z} - d) < 3.0 ? 1.0 : 0.25, sqrt({z} - d) >= 3.0 ? 1.0 : 0.5, sqrt({z} - d) == sqrt({z} - d) ? 0.75 : 0.125, "
               "(!(sqrt({z} - d) > 1.0) && (d != {z} || d <= 1.0)) ? 1.0 : 0.0)",
    "rounding": "vec4(ceil(d * 0.01) * 0.1, trunc(-d * 0.013) * -0.1, fract(-d * 0.037), abs(sign(d - {z}) * 0.5 - floor(d * 0.002)))",
    "mix_swizzle": "mix(vec4(d * 0.001, 0.2, 0.3, 1.0), (#e6331a80 * vec4(1.0, d * 0.002, 1.0, 1.0)).wzyx, clamp(d / 300.0, 0.0, 1.0)).bgra",
    "alpha_toggle": "vec4(0.8, 0.3, mod(d, 3.0) / 3.0, mod(d, 2.0) < 1.0 ? 1.0 : 0.5)",
}
# 64 instructions with all 8 registers live (an EdgeGen expression; test_color_programs.py checks both limits)
LIMIT = ("mix((vec4(vec2(1, 2.1), vec2(0.65, d)) * exp2((1.0 / (d - {z})))), mix(vec4(vec2(0.1, 0.18), vec2(0.97, d)), "
         "mix(#c13bb3, vec4(4, 4, d, 1.65), float(d)), float(log2(float(3)))), float(((((2.3 < 0.1 && 0.453 >= 1) || !(8 > 2)) "
         "? float(0.453) : float(8)) / (abs(mod(float(d), 1.75)) + 0.5))))")
LIMITS = {"limit": LIMIT}


class EdgeGen(_Gen):
    """_Gen's expressions plus the transcendentals and the edge operands of PROGRAMS"""

    EDGE = ["(1.0 / (d - {z}))", "(0.0 * (1.0 / (d - {z})))", "exp(d)", "exp(-d)", "sqrt({z} - d)", "(-0.0 * d)",
            "(d * 1e6)", "(d * 1e9)"]

    def __init__(self, rng, z):
        super().__init__(rng)
        self.z = z

    def scalar(self, depth):
        if depth > 0 and self.r.random() < 0.35:
            a = self.scalar(depth - 1)
            e = self.r.choice(self.EDGE).format(z=self.z) if self.r.random() < 0.5 else self.fl(a)
            k = self.r.integers(0, 9)
            fn = ["sin", "cos", "tan", "log", "log2", "exp", "exp2", "sqrt", "atan"][k]
            if fn == "atan" and self.r.random() < 0.5:
                return f"atan({e}, {self.fl(self.scalar(depth - 1))})"
            if self.r.random() < 0.2:
                return f"pow({e}, {self.fl(a)})"
            return f"{fn}({e})"
        return super().scalar(depth)


def program_text(name, module):
    z = {"bars": "40.5", "graph": "40.0"}.get(module, "40.25")
    text = PROGRAMS.get(name) or LIMITS.get(name)
    return text.format(z=z)


_compiled = {}


def compile_expr(module, color, outline=None):
    """the colour / outline fields load_config makes of `#define COLOR color` (and BAR_OUTLINE) for `module`"""
    key = (module, color, outline)
    if key not in _compiled:
        with tempfile.TemporaryDirectory() as d:
            with open(os.path.join(d, "rc.glsl"), "w") as f:
                f.write(f"#request mod {module}\n")
            with open(os.path.join(d, module + ".glsl"), "w") as f:
                f.write(f"#define COLOR {color}\n" + (f"#define BAR_OUTLINE {outline}\n" if outline else ""))
            _compiled[key] = g.load_config([d])
    return _compiled[key]


def params(module, w, h, color, outline=None, **over):
    """default parameters of `module` at w x h with the compiled COLOR (and BAR_OUTLINE) programs and the overrides"""
    src = compile_expr(module, color, outline)
    p = g.default_params(module, n=N, w=w, h=h, **over)
    setattr(p, f"{module}_color", getattr(src, f"{module}_color"))
    setattr(p, f"{module}_color_prog", getattr(src, f"{module}_color_prog"))
    if module == "bars" and outline:
        p.bars_outline_mode = src.bars_outline_mode
        p.bars_outline_prog = src.bars_outline_prog
        p.bars_outline[:] = list(src.bars_outline)
    return p


def prog_of(p, outline=False):
    m = g.MODULES[p.module]
    return p.bars_outline_prog if outline else getattr(p, f"{m}_color_prog")


def opcodes(prog):
    return {OPS[prog.ops[i].op] for i in range(prog.n_ops)}


def registers(prog):
    return {r for i in range(prog.n_ops) for r in (prog.ops[i].dst,)}


# ---- styles mixed in one batch: slot 0, AMPLIFY only (the program is kept), bg only (the bars outline becomes a constant,
# COLOR stays a program), fg + bg (the program is dropped) -----------------------------------------------------------------
AMP = dict(bars="bars_amplify", radial="radial_amplify", graph="graph_vscale")
BG = (0.4, 0.5, 0.1, 1.0)
FG = (0.2, 0.9, 0.4, 0.8)


def styles_for(p):
    a = getattr(p, AMP[g.MODULES[p.module]])
    return [None, {"amplify": 0.8 * a}, {"bg": BG}, {"fg": FG, "bg": BG}]


# ---- sites ------------------------------------------------------------------------------------------------------------
BLEND = dict(premultiply_alpha=0, clear_color=[0.05, 0.1, 0.15, 1.0])
EVERY = tuple(PROGRAMS) + tuple(LIMITS)
HD_RADIAL = ("log_domain", "trig_large", "atan_quadrants", "nan_cmp")


def _bars(w, h, **over):
    return dict(dict(bars_amplify=1.25 * h, bars_outline_width=1.0), **over)


def _graph(w, h, **over):
    return dict(dict(graph_vscale=1.25 * h), **over)


def _radial(w, h, **over):
    base = dict(radial_radius=30.0, radial_amplify=50.0) if h < 1080 else {}
    base.update(over)
    return base


# (name, module, w, h, programs, overrides, environment, styled)
SITES = [
    ("bars-1920x1080", "bars", 1920, 1080, EVERY, _bars(1920, 1080), {}, True),
    ("bars-blend-1920x1080", "bars", 1920, 1080, ("inf_nan", "log_domain", "nan_cmp", "alpha_toggle"), _bars(1920, 1080, **BLEND), {}, True),
    ("bars-256x16384", "bars", 256, 16384, ("trig_large", "log_domain"), _bars(256, 16384), {}, True),
    ("bars-333x181", "bars", 333, 181, EVERY, _bars(333, 181), {}, True),                     # w % 4 != 0: generic
    ("bars-blend-333x181", "bars", 333, 181, EVERY, _bars(333, 181, **BLEND), {}, True),
    ("bars-mirror-180x332", "bars", 180, 332, ("inf_nan", "trig_large", "nan_cmp"), _bars(180, 332, bars_mirror_yx=1,
                                                                                           bars_amplify=1.25 * 180), {}, True),
    ("graph-1920x1080", "graph", 1920, 1080, EVERY, _graph(1920, 1080), {}, True),
    ("graph-nocoltab-1920x1080", "graph", 1920, 1080, ("alpha_toggle", "inf_nan", "nan_cmp"), _graph(1920, 1080),
     dict(NO_COLTAB=1), True),
    ("graph-blend-332x181", "graph", 332, 181, EVERY, _graph(332, 181, **BLEND), {}, True),
    ("graph-blend-nocoltab-332x181", "graph", 332, 181, ("alpha_toggle", "log_domain"), _graph(332, 181, **BLEND),
     dict(NO_COLTAB=1), True),
    ("graph-invert-332x181", "graph", 332, 181, ("alpha_toggle", "inf_nan"), _graph(332, 181, graph_invert=1), {}, True),
    ("radial-1920x1080", "radial", 1920, 1080, HD_RADIAL, _radial(1920, 1080), {}, True),
    ("radial-3840x2160", "radial", 3840, 2160, ("trig_large",), _radial(3840, 2160), {}, True),
    ("radial-332x181", "radial", 332, 181, EVERY, _radial(332, 181), {}, True),
    ("radial-blend-332x181", "radial", 332, 181, EVERY, _radial(332, 181, **BLEND), {}, True),
    ("radial-nogeo-332x181", "radial", 332, 181, EVERY, _radial(332, 181), dict(NO_GEO=1), True),
    ("radial-nogeo-blend-332x181", "radial", 332, 181, ("log_domain", "nan_cmp"), _radial(332, 181, **BLEND),
     dict(NO_GEO=1), True),
    ("radial-outline-332x181", "radial", 332, 181, ("atan_quadrants", "sqrt_pow"), _radial(332, 181, radial_bar_outline_width=2.0),
     {}, True),
    ("radial-outline-blend-332x181", "radial", 332, 181, ("mod_smooth",), _radial(332, 181, radial_bar_outline_width=2.0, **BLEND),
     {}, True),
]
# bars BAR_OUTLINE: the program after `name` in EVERY, so each program also runs as an outline
def outline_for(name):
    return EVERY[(EVERY.index(name) + 1) % len(EVERY)]


def cases():
    """[(case id, site, program name, params)]"""
    out = []
    for site in SITES:
        name, module, w, h, progs, over, env, styled = site
        for prog in progs:
            outline = program_text(outline_for(prog), module) if module == "bars" else None
            out.append((f"{name}-{prog}", site, prog, params(module, w, h, program_text(prog, module), outline, **over)))
    return out


# ---- the reference's own frames on Mesa llvmpipe (tests/golden/make_color_expr_llvmpipe_golden.py) ---------------------
LLVMPIPE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "color_expr_llvmpipe.npz")
FLIP_PIXELS = 8          # hard-edge pixels off by more than 1 LSB per case, as tests/test_llvmpipe_golden.py
# Where llvmpipe leaves IEEE, the VM keeps its rules (DESIGN §4.5) and the pixels that differ by more than 1 LSB are
# counted here, case by case, with what llvmpipe does there:
LLVMPIPE_DIFFERS = {
    "inf_nan": "on the row d = Z llvmpipe gives 0 * (1 / 0) = 0, not NaN, and stores +inf as 0",
    "log_domain": "rows d >= 88.5: llvmpipe's log(exp(d)) stays finite (about 88.7) and log(exp(-d)) differs on subnormals",
    "sqrt_pow": "llvmpipe's pow(x, 0.5) for x < 0 gives pow(|x|, 0.5), not NaN",
    "trig_large": "llvmpipe's sin / cos / tan of d * 1e3 .. d * 1e9 differ from the exactly reduced values on every row",
    "mod_smooth": "llvmpipe's mod(x, 0.0) gives x, not NaN",
    "nan_cmp": "on rows where sqrt(Z - d) is NaN, llvmpipe's comparisons and `!` do not give IEEE's answers",
}
LLVMPIPE_COUNTS = {"bars_inf_nan": 225, "graph_inf_nan": 166, "bars_log_domain": 180, "graph_log_domain": 171,
                   "radial_log_domain": 29, "bars_sqrt_pow": 19265, "graph_sqrt_pow": 20745, "radial_sqrt_pow": 7938,
                   "bars_trig_large": 23650, "graph_trig_large": 26004, "radial_trig_large": 18486, "bars_mod_smooth": 23735,
                   "graph_mod_smooth": 28239, "radial_mod_smooth": 16792, "bars_nan_cmp": 5180, "graph_nan_cmp": 6973,
                   "radial_nan_cmp": 4032}
EXACT_EXPRS = ("rounding",)      # no transcendental: every operation exactly rounded in both


def llvmpipe_names():
    return [str(c) for c in np.load(LLVMPIPE)["case_names"]]


def llvmpipe_case(name):
    """(params, [2][n] textures, llvmpipe's frame) of one case; frames are row 0 = bottom, as the product's"""
    import json
    from glava_b200.api import Params
    z = np.load(LLVMPIPE)
    return Params.from_dict(json.loads(str(z[f"{name}_params"]))), z[f"{name}_tex"], z[f"{name}_frame"]


def host_frame(p, tl, tr):
    """emul.raster of (p, tl, tr), radial through the geometry helper, bars / graph through the row tables"""
    from tests import emul
    if g.MODULES[p.module] == "radial":
        return emul.RadialGeo(p).frame(tl, tr)
    return emul.raster(p, tl, tr, fast=not p.bars_mirror_yx)


def check_against_llvmpipe(name, got, want):
    d = np.abs(got.astype(int) - want.astype(int)).max(axis=2)
    off, bad = int((d > 0).sum()), int((d > 1).sum())
    expr = name.split("_", 1)[1]
    if expr in EXACT_EXPRS and g.MODULES.index(name.split("_")[0]) != g.MODULES.index("radial"):
        assert off == 0, (name, "exactly rounded expression: pixels differ", off)
    assert bad <= FLIP_PIXELS + LLVMPIPE_COUNTS.get(name, 0), (name, off, bad, LLVMPIPE_DIFFERS.get(expr))
    return off, bad
