"""CPU tier for the colour-expression programs (tests/color_programs.py): the colour VM (raster_core.h eval_color_prog,
through the host build) against a float64 reference interpreter, its special-value rules, constant folding and the
hoisted row tables against per-pixel evaluation, plus the coverage the case list claims.  GPU tier:
tests/test_gpu_color_programs.py."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import glava_b200 as g
from glava_b200 import api
from tests import color_programs as cp
from tests import emul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
OP = {name: k for k, name in enumerate(cp.OPS)}
INF, NAN = float("inf"), float("nan")


# ---- float64 reference interpreter of glava_b200_color_prog ----------------------------------------------------------
def f32(v):
    return float(F32(v))


def _div(a, b):
    if b == 0.0:
        return NAN if a == 0.0 or a != a else math.copysign(INF, a) * math.copysign(1.0, b)
    return f32(a / b)


def _mul(a, b):
    return f32(a * b) if not ((a == 0.0 and math.isinf(b)) or (b == 0.0 and math.isinf(a))) else NAN


def _add(a, b):
    return f32(a + b) if not (math.isinf(a) and math.isinf(b) and a != b) else NAN


def _log(x):                           # IEEE: -inf at +-0, NaN below 0 and at NaN, +inf at +inf
    if x != x or x < 0:
        return NAN
    return -INF if x == 0 else (INF if math.isinf(x) else math.log(x))


def _exp(x):
    if x != x:
        return NAN
    return 0.0 if x == -INF else (INF if x > 709 else math.exp(x))


def _pow(x, y):                        # 0^y = 0 for y > 0 (else NaN); x^y = exp(y log x) otherwise
    if x == 0.0:
        return 0.0 if y > 0 else NAN
    lg = _log(x)
    return _exp(_mul(y, lg) if math.isinf(lg) else y * lg)


def _trig(fn, x):
    return NAN if not math.isfinite(x) else fn(x)


def _atan2(y, x):                      # atan(0, 0) := 0 for either sign of x (raster_core.h cvm_atan2 / glm_atan2)
    if x == 0.0 and y == 0.0:
        return math.copysign(0.0, y)
    return math.atan2(y, x)


def _floor(v):
    return float(np.floor(v))


def _ceil(v):
    return float(np.ceil(v))


def _trunc(v):
    return float(np.trunc(v))


def _clamp(v, lo, hi):                 # g_clamp / g_min(g_max()): the comparisons decide, NaN falls through
    return lo if v < lo else (hi if v > hi else v)


def _smooth(e0, e1, x):
    t = _clamp(_div(f32(x - e0) if not (math.isinf(x) and math.isinf(e0) and x == e0) else NAN,
                    f32(e1 - e0) if not (math.isinf(e1) and math.isinf(e0) and e1 == e0) else NAN), 0.0, 1.0)
    return _mul(_mul(t, t), f32(3.0 - _mul(2.0, t)))


EXACT1 = {"NEG": lambda v: -v, "ABS": abs, "FLOOR": _floor, "CEIL": _ceil, "FRACT": lambda v: _add(v, -_floor(v)),
          "SQRT": lambda v: NAN if v < 0 else (v if v == 0 or v != v else f32(math.sqrt(v))),
          "SIGN": lambda v: 1.0 if v > 0 else (-1.0 if v < 0 else 0.0), "TRUNC": _trunc,
          "NOT": lambda v: 0.0 if v != 0.0 else 1.0}
EXACT2 = {"ADD": _add, "SUB": lambda a, b: _add(a, -b) if b == b else NAN, "MUL": _mul, "DIV": _div,
          "MIN": lambda a, b: b if b < a else a, "MAX": lambda a, b: b if a < b else a,
          "MOD": lambda a, b: _add(a, -_mul(b, _floor(_div(a, b)))), "STEP": lambda a, b: 0.0 if b < a else 1.0,
          "LT": lambda a, b: float(a < b), "LE": lambda a, b: float(a <= b), "EQ": lambda a, b: float(a == b),
          "NE": lambda a, b: float(a != b), "AND": lambda a, b: float(a != 0.0 and b != 0.0),
          "OR": lambda a, b: float(a != 0.0 or b != 0.0)}
EXACT3 = {"MIX": lambda a, b, c: _add(_mul(a, f32(1.0 - c) if math.isfinite(c) else (NAN if c != c else -c)), _mul(b, c)),
          "CLAMP": lambda a, b, c: (lambda m: c if c < m else m)(b if a < b else a), "SMOOTHSTEP": _smooth,
          "SELECT": lambda a, b, c: a if c != 0.0 else b}
# transcendentals: the exact value (float64) of the operation on the float32 operands
TRANS1 = {"SIN": lambda v: _trig(math.sin, v), "COS": lambda v: _trig(math.cos, v), "TAN": lambda v: _trig(math.tan, v),
          "LOG": _log, "LOG2": lambda v: _log(v) / math.log(2) if math.isfinite(_log(v)) else _log(v), "EXP": _exp,
          "EXP2": lambda v: NAN if v != v else (0.0 if v == -INF else (INF if v > 1000 else 2.0 ** v))}
TRANS2 = {"POW": _pow, "ATAN2": _atan2}


def reference(prog, x, exact_trans=False):
    """float64 interpretation of a colour program at X: every exactly rounded operation rounded to float32 as the VM does,
    the transcendentals exact (exact_trans=False: rounded to float32, which is what an ulp comparison starts from)"""
    reg = [[0.0] * 4 for _ in range(8)]
    for i in range(prog.n_ops):
        o = prog.ops[i]
        name, dst, a, b, imm = cp.OPS[o.op], o.dst & 7, o.a & 7, o.b & 7, float(o.imm)
        A, B = reg[a], reg[b]
        Cc = reg[int(imm) & 7] if name in EXACT3 else None
        if name == "SPLAT":
            reg[dst] = [imm] * 4
        elif name == "VAR":
            reg[dst] = [x] * 4
        elif name == "LANE":
            reg[dst] = list(reg[dst]); reg[dst][a & 3] = imm
        elif name == "SHUF":
            R = list(reg[dst])
            for k in range(4):
                sel = (int(imm) >> (3 * k)) & 7
                if sel < 4:
                    R[k] = A[sel]
            reg[dst] = R
        elif name in EXACT1:
            reg[dst] = [EXACT1[name](v) for v in A]
        elif name in EXACT2:
            reg[dst] = [EXACT2[name](v, w) for v, w in zip(A, B)]
        elif name in EXACT3:
            reg[dst] = [EXACT3[name](v, w, u) for v, w, u in zip(A, B, Cc)]
        elif name in TRANS1:
            reg[dst] = [TRANS1[name](v) if exact_trans else f32(TRANS1[name](v)) for v in A]
        else:
            reg[dst] = [TRANS2[name](v, w) if exact_trans else f32(TRANS2[name](v, w)) for v, w in zip(A, B)]
        reg[dst] = [float(v) for v in reg[dst]]
    return reg[prog.result & 7]


def same_bits(a, b):
    """float32 equality with NaN == NaN (any payload: unorm8 and every VM operation treat them alike) and -0 != +0"""
    a, b = F32(a), F32(b)
    return (a != a and b != b) or a.view(np.uint32) == b.view(np.uint32)


# ---- operands: dense grids, the whole finite range and every special value --------------------------------------------
def specials():
    fi = np.finfo(np.float32)
    base = [0.0, 1.0, 0.5, 2.0, 3.0, 1e-3, 0.75, 1.5, math.pi / 2, math.pi, 40.5, 8192.0, 8192.5, 3.3e9, 4e9, 1e10, 1e20,
            float(fi.tiny), float(fi.smallest_subnormal), 1e-40, 1e-45, float(fi.max), 88.7, 88.8, 103.0, 104.0, 150.0, 2.0 ** 31,
            2.0 ** 31 * math.pi / 2, 1e38, INF]
    out = [f32(v) for v in base] + [-f32(v) for v in base] + [NAN]
    return out


def operands(seed, n):
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 0x7f800000, n, dtype=np.int64).astype(np.uint32).view(np.float32)     # the whole finite range
    sign = np.where(rng.random(n) < 0.5, -1, 1).astype(np.float32)
    grid = np.concatenate([np.linspace(-20, 20, n // 2), np.linspace(-1e4, 1e4, n // 4), np.geomspace(1e-30, 1e30, n // 4)])
    return [float(v) for v in np.concatenate([bits * sign, grid.astype(np.float32)])] + specials()


def one_op(name, imm=0):
    """reg0 = X, reg1 = the second operand, reg2 = the third: dst 3 = op(reg0, reg1 [, reg2])"""
    prog = api.ColorProg()
    ops = [(OP["VAR"], 0, 0, 0, 0.0), (OP["SPLAT"], 1, 0, 0, 0.0), (OP["SPLAT"], 2, 0, 0, 0.0), (OP[name], 3, 0, 1, 2.0)]
    for k, o in enumerate(ops):
        prog.ops[k].op, prog.ops[k].dst, prog.ops[k].a, prog.ops[k].b, prog.ops[k].imm = o
    prog.n_ops, prog.result = len(ops), 3
    return prog


def run(prog, x, y=0.0, z=0.0):
    prog.ops[1].imm, prog.ops[2].imm = y, z
    return emul.eval_color(prog, x)[0]


SECOND = [0.0, -0.0, 1.0, -1.0, 0.5, 1.75, 3.0, -2.5, 1e-40, 1e30, INF, -INF, NAN]


@pytest.mark.parametrize("name", sorted(EXACT1) + sorted(EXACT2) + sorted(EXACT3))
def test_exactly_rounded_ops_match_float64_bit_for_bit(name, built):
    prog = one_op(name)
    xs = operands(OP[name], 600)
    ys = SECOND if name not in EXACT1 else [0.0]
    zs = [0.0, 1.0, 0.25, NAN, INF, -0.0] if name in EXACT3 else [0.0]
    bad = []
    for x in xs:
        for y in ys:
            for z in zs:
                got = run(prog, x, y, z)
                want = reference(prog, float(F32(x)))[0]
                if not same_bits(got, want):
                    bad.append((x, y, z, float(got), want))
    assert not bad, (name, len(bad), bad[:5])


def _ulps(got, want):
    w = F32(want)
    if not np.isfinite(w):
        return 0.0 if same_bits(got, w) else INF
    return abs(float(got) - want) / float(np.spacing(max(abs(w), np.finfo(np.float32).tiny)))


# stated bounds, in ulps of the float32 result, over the whole finite range (the sin / cos / tan bound is absolute near
# their zeros: 2^-24 / 2^-22, what the reductions promise there)
ULP = {"SIN": 2.0, "COS": 2.0, "TAN": 4.0, "LOG": 2.0, "LOG2": 3.0, "EXP": 1.0, "EXP2": 1.0, "ATAN2": 3.0}
ABS = {"SIN": 2.0 ** -24, "COS": 2.0 ** -24, "TAN": 2.0 ** -22}


@pytest.mark.parametrize("name", sorted(TRANS1) + ["ATAN2"])
def test_transcendentals_within_their_ulp_bounds_over_the_whole_range(name, built):
    prog = one_op(name)
    xs = operands(100 + OP[name], 4000)
    ys = [1.0, -1.0, 0.5, -3.0, 1e-30, 1e30, 0.0, -0.0] if name == "ATAN2" else [0.0]
    worst, at = 0.0, None
    for x in xs:
        for y in ys:
            got = run(prog, x, y)
            prog.ops[1].imm = y
            want = reference(prog, float(F32(x)), exact_trans=True)[0]
            if want != want:
                assert got != got, (name, x, y, float(got))
                continue
            if name in ("SIN", "COS", "TAN") and math.isfinite(x) and name != "TAN":
                assert -1.0 <= got <= 1.0, (name, x, float(got))
            if abs(want) < 2.0 ** -126 and want != 0.0:
                continue                                  # subnormal results: the absolute error is below the smallest normal
            u = _ulps(got, want)
            if name in ABS and abs(float(got) - want) <= ABS[name]:
                u = min(u, 0.0)
            if u > worst:
                worst, at = u, (x, y, float(got), want)
    assert worst <= ULP[name], (name, worst, at)


def test_pow_within_bounds_and_its_domain(built):
    prog = one_op("POW")
    worst = 0.0
    for x in operands(7, 1500):
        for y in (2.5, 0.5, -1.0, 2.0, 0.0, 1e-3):
            got = run(prog, x, y)
            prog.ops[1].imm = y
            want = reference(prog, float(F32(x)), exact_trans=True)[0]
            if want != want:
                assert got != got, (x, y, float(got))
            elif abs(want) > 2.0 ** -126 and abs(want) < 3e38 and abs(y * math.log(abs(x))) < 80:
                worst = max(worst, _ulps(got, want) / max(1.0, abs(y * math.log(abs(x)))))
            elif not math.isfinite(want):
                assert float(got) == want, (x, y, float(got), want)
    assert worst <= 2.0, worst                             # exp(y log x): the log's error scaled by |y log x|


@pytest.mark.parametrize("name,x,y,want", [
    ("LOG", -4.0, 0, NAN), ("LOG", -1e-3, 0, NAN), ("LOG", 0.0, 0, -INF), ("LOG", -0.0, 0, -INF), ("LOG", INF, 0, INF),
    ("LOG", NAN, 0, NAN), ("LOG", 1e-40, 0, math.log(f32(1e-40))), ("LOG", 1e-45, 0, math.log(f32(1e-45))),
    ("LOG2", -4.0, 0, NAN), ("LOG2", 0.0, 0, -INF), ("LOG2", INF, 0, INF), ("LOG2", 1e-40, 0, math.log2(f32(1e-40))),
    ("POW", -4.0, 0.5, NAN), ("POW", NAN, 2.0, NAN), ("POW", -4.0, 2.0, NAN), ("POW", 1e-40, 0.5, math.sqrt(f32(1e-40))),
    ("POW", INF, 2.0, INF), ("POW", INF, -1.0, 0.0), ("POW", 0.0, 2.0, 0.0),
    ("SIN", 3.3e9, 0, math.sin(f32(3.3e9))), ("SIN", 4e9, 0, math.sin(f32(4e9))), ("SIN", 1e10, 0, math.sin(f32(1e10))),
    ("SIN", 1e20, 0, math.sin(f32(1e20))), ("SIN", -1e20, 0, math.sin(f32(-1e20))), ("SIN", 3.4028235e38, 0, math.sin(f32(3.4028235e38))),
    ("COS", 1e10, 0, math.cos(f32(1e10))), ("COS", 8193.0, 0, math.cos(8193.0)), ("TAN", 1e20, 0, math.tan(f32(1e20))),
    ("SIN", INF, 0, NAN), ("COS", -INF, 0, NAN), ("TAN", NAN, 0, NAN),
    ("ATAN2", INF, INF, math.pi / 4), ("ATAN2", INF, -INF, 3 * math.pi / 4), ("ATAN2", -INF, INF, -math.pi / 4),
    ("ATAN2", -INF, -INF, -3 * math.pi / 4), ("ATAN2", 0.0, -1.0, math.pi), ("ATAN2", -0.0, -1.0, -math.pi),
    ("ATAN2", INF, 1.0, math.pi / 2), ("ATAN2", 1.0, -INF, math.pi), ("ATAN2", 0.0, 0.0, 0.0),
])
def test_special_value_rules(name, x, y, want, built):
    """DESIGN §4.5's table of the VM's answers at the domain edges"""
    got = float(run(one_op(name), x, y))
    if want != want:
        assert got != got, (name, x, y, got)
    elif math.isinf(want):
        assert got == want, (name, x, y, got)
    else:
        assert abs(got - want) <= 3 * float(np.spacing(F32(abs(want)))) + (2.0 ** -24 if name in ("SIN", "COS", "TAN") else 0), \
            (name, x, y, got, want)


def _same_class(got, want):
    """a program with transcendentals against the reference with float32-rounded transcendentals: NaN in the same lanes,
    the same infinities, and finite lanes within 1e-4 relative (or 1e-6 absolute; a few ulps carried through the program)"""
    got = float(got)
    if want != want or got != got:
        return want != want and got != got
    if math.isinf(want) or math.isinf(got):
        return got == want
    return abs(got - want) <= max(1e-6, 1e-4 * abs(want))


def test_programs_match_the_reference_interpreter(built):
    """whole programs: exactly rounded ones bit for bit at every operand; programs with transcendentals agree where the
    reference's float32-rounded transcendentals meet the VM's (the VM is within the ulp bounds above)"""
    xs = [float(v) for v in np.concatenate([np.arange(0.5, 200, 1.0), np.arange(3390.5, 3420, 1.0), [16383.5, 1e5, -3.5]])]
    for name in cp.EVERY:
        for module in ("bars", "graph"):
            p = cp.params(module, 64, 64, cp.program_text(name, module))
            prog = cp.prog_of(p)
            exact = not (cp.opcodes(prog) & set(TRANS1) | cp.opcodes(prog) & set(TRANS2))
            for x in xs:
                got, want = emul.eval_color(prog, x), reference(prog, x)
                if exact:
                    assert all(same_bits(a, b) for a, b in zip(got, want)), (name, module, x, got, want)
                else:
                    for a, b in zip(got, want):
                        assert _same_class(a, b), (name, module, x, got, want)


def test_random_edge_programs_match_the_reference_interpreter(built):
    """EdgeGen's programs (transcendentals and edge operands): the exactly rounded ones bit for bit; the others in the same
    class as the reference with float32-rounded transcendentals (_same_class)"""
    rng = np.random.default_rng(20261017)
    gen = cp.EdgeGen(rng, "40.5")
    xs = [0.5, 1.5, 40.5, 41.5, 87.5, 95.5, 104.5, 1000.5, 3400.5, 16383.5]
    checked = exact_checked = 0
    for i in range(150):
        expr = gen.vec(4, int(rng.integers(1, 4)))
        try:
            p = cp.compile_expr("bars", expr)
        except g.GlavaError as e:
            assert "more than 8 live" in str(e) or "longer than 64" in str(e), (expr, str(e))
            continue
        if p.bars_color.mode != 2:
            continue
        prog = p.bars_color_prog
        trans = cp.opcodes(prog) & (set(TRANS1) | set(TRANS2))
        for x in xs:
            got, want = emul.eval_color(prog, x), reference(prog, x)
            if not trans:
                assert all(same_bits(a, b) for a, b in zip(got, want)), (expr, x, got, want)
            else:
                assert all(_same_class(a, b) for a, b in zip(got, want)), (expr, x, got, want)
        checked += 1
        exact_checked += not trans
    assert checked >= 100 and exact_checked >= 20, (checked, exact_checked)


# ---- coverage of the case list ---------------------------------------------------------------------------------------
def test_cases_reach_every_opcode_and_the_limits(built):
    color, outline = set(), set()
    for _, site, name, p in cp.cases():
        color |= cp.opcodes(cp.prog_of(p))
        if site[1] == "bars":
            assert p.bars_outline_mode == 2
            outline |= cp.opcodes(cp.prog_of(p, outline=True))
    assert color == set(cp.OPS), sorted(set(cp.OPS) - color)
    assert outline == set(cp.OPS), sorted(set(cp.OPS) - outline)
    lim = cp.prog_of(cp.params("bars", 64, 64, cp.program_text("limit", "bars")))
    assert lim.n_ops == 64 and max(cp.registers(lim)) == 7
    # the graph program whose alpha toggles between 1 and < 1 from row to row (the row table's "rows y-1, y, y+1 opaque")
    tog = cp.prog_of(cp.params("graph", 64, 64, cp.program_text("alpha_toggle", "graph")))
    alpha = [float(emul.eval_color(tog, float(y))[3]) for y in range(8)]
    assert alpha == [1.0, 0.5] * 4, alpha


def _slots(p, styles):
    sp = [p]
    for s in styles:
        if s is not None:
            sp.append(g.style_params(p, s))
    pairs = {(None if s is None else (str(s.get("fg")), str(s.get("bg")))) for s in styles}
    return sp, len(pairs)


def test_cases_select_every_kernel_form(tmp_path_factory, built):
    from tests.test_stream_styles import styled_plan
    seen = set()
    for _, site, name, p in cp.cases():
        _, module, w, h, _, over, env, styled = site
        plain = emul.raster_plan(p, 8, 8, env)["kernel"]
        seen.add((module, plain, p.premultiply_alpha != 0, False))
        sp, caches = _slots(p, cp.styles_for(p))
        plan = styled_plan(tmp_path_factory, sp, caches, 8, 8, env)
        assert plan["styled"] == 1
        seen.add((module, plan["kernel"], p.premultiply_alpha != 0, True))
    # native: the row tables (bars, graph with and without the column table: graph_tab4 / graph), the radial cache and
    # the per-pixel kernels; premultiply_alpha = 0 runs every module through the generic kernel's blended form
    forms = [("bars", "bars", True), ("bars", "generic", True), ("graph", "graph_tab4", True), ("graph", "graph", True),
             ("radial", "radial_geo", True), ("radial", "radial", True), ("bars", "generic", False), ("graph", "generic", False),
             ("radial", "generic", False)]
    want = {f + (styled,) for f in forms for styled in (False, True)}
    assert want <= seen, sorted(want - seen)


# ---- folding, hoisting ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", cp.EVERY)
def test_constant_folding_agrees_with_the_program(name, built):
    """the expression with `d` spelled as a literal folds at config time (mode 1) to what the program gives at that d"""
    text = cp.program_text(name, "bars")
    prog = cp.prog_of(cp.params("bars", 64, 64, text))
    for x in (0.5, 40.5, 87.5, 100.5, 3400.5, 16383.5):
        folded = cp.compile_expr("bars", re.sub(r"\bd\b", "(%r)" % x, text))
        assert folded.bars_color.mode == 1, (name, x)
        got = list(folded.bars_color.lo)
        want = emul.eval_color(prog, x)
        assert all(same_bits(a, b) for a, b in zip(got, want)), (name, x, got, want)


def _band(p, tl, tr, y0, y1):
    out = np.zeros((p.h, p.w, 4), np.uint8)
    emul.lib().emul_raster(C.addressof(p), tl.ctypes.data, tr.ctypes.data, out.ctypes.data, y0, y1)
    return out[y0:y1]


def test_hoisted_rows_equal_per_pixel_evaluation(built):
    """every bars and graph case: the row-table evaluation (emul.raster fast=True, as the kernels) equals per-pixel
    evaluation (the generic kernel's) on rows that reach the programs' edges"""
    from tests import test_gpu_raster_variants as rv
    rows = rv._edges(cp.N)
    ramp = np.linspace(0, 65535, cp.N).round().astype(np.uint16)
    rows.append((ramp, ramp[::-1].copy()))
    for cid, site, name, p in cp.cases():
        if site[1] not in ("bars", "graph") or p.bars_mirror_yx:
            continue
        bands = [(0, min(p.h, 120))] + ([(3390, 3420), (p.h - 20, p.h)] if p.h > 3420 else [])
        for tl, tr in rows[1:]:
            fast = emul.raster(p, tl, tr, fast=True)
            for y0, y1 in bands:
                assert np.array_equal(fast[y0:y1], _band(p, tl, tr, y0, y1)), (cid, y0, y1)


def test_gpu_script_passes_its_dry_run(built):
    """tests/test_gpu_color_programs.py on small cases against the emulation-backed renderer of tools/dryrun_gpu_tests.py"""
    ids = ["test_programs_on_the_device[bars-333x181-inf_nan]", "test_programs_on_the_device[graph-blend-332x181-alpha_toggle]",
           "test_programs_on_the_device[radial-nogeo-332x181-log_domain]", "test_programs_on_the_device[radial-outline-332x181-sqrt_pow]",
           "test_reconfigure_swaps_programs_with_live_marks"]
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dryrun_gpu_tests.py")] +
                         [f"tests/test_gpu_color_programs.py::{i}" for i in ids], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert f"{len(ids)} passed" in out.stdout and "failed" not in out.stdout


@pytest.mark.parametrize("name", cp.llvmpipe_names())
def test_llvmpipe_frames_replayed_through_the_host_build(name, built):
    """the reference's own shaders on Mesa llvmpipe: <= 1 LSB plus a handful of hard-edge pixels, the exactly rounded
    expression bit for bit (bars, graph), and the pixels where llvmpipe leaves IEEE counted (color_programs.LLVMPIPE_DIFFERS)"""
    p, tex, want = cp.llvmpipe_case(name)
    assert want.any()
    cp.check_against_llvmpipe(name, cp.host_frame(p, tex[0], tex[1]), want)


@pytest.mark.parametrize("cid", [c[0] for c in cp.cases() if c[1][1] == "radial" and c[1][2] < 1000])
def test_radial_geometry_helper_equals_per_pixel_raster(cid, built):
    """emul.RadialGeo (the radial reference of the GPU tests) against emul.raster's per-pixel radial_px"""
    from tests import test_gpu_raster_variants as rv
    _, site, name, p = next(c for c in cp.cases() if c[0] == cid)
    tl, tr = rv._stack(rv._edges(cp.N) + rv._polar_bands(cp.N, p.w + p.h))
    geo = emul.RadialGeo(p)
    for s in range(tl.shape[0]):
        assert np.array_equal(geo.frame(tl[s], tr[s]), emul.raster(p, tl[s], tr[s])), (cid, s)
