"""Expression strings (dig_b200/basis.py) -> sm_90a device code with ATen-CUDA rounding.

The reference evaluates each closed form through ``sympy.lambdify`` with torch functions, i.e.
Python walks the expression and every arithmetic node becomes ONE ATen elementwise kernel on
fp32 tensors (reference spherenet/features.py:200-222,240-263).  To reproduce those bits inside
a fused kernel this generator parses the same source string with ``ast`` and emits one explicit
correctly-rounded fp32 intrinsic per node (`__fmul_rn`, `__fadd_rn`, ... are never contracted
into FMAs by nvcc), following the scalar/tensor typing rules of torch:

  * python-scalar (op) python-scalar is folded in double precision, as Python does;
  * tensor (op) python-scalar rounds the scalar to fp32 first (ATen wraps it as opmath_t=float);
  * ``t ** 2 -> t*t``, ``t ** 3 -> (t*t)*t``, ``t ** 0.5 -> sqrtf``, other exponents -> powf
    (ATen pow_tensor_scalar special cases);
  * ``t / c`` is ``t * (1.0f / c)`` on CUDA (ATen div_true_kernel_cuda's CPU-scalar fast path);
  * ``c / t`` is ``reciprocal(t) * c`` (torch.Tensor.__rtruediv__);
  * sin / cos / sqrt map to the precise libdevice sinf / cosf / sqrtf (no fast-math).

Identical sub-expressions are emitted once (they are pure, so this is exact).
"""
import ast
import math

import numpy as np


def f32_literal(v):
    f = np.float32(v)
    if not np.isfinite(f):
        raise ValueError(v)
    s = "%.9g" % float(f)
    if "." not in s and "e" not in s and "n" not in s:
        s += ".0"
    return s + "f"


class _Emitter:
    def __init__(self, var_names):
        self.lines = []
        self.cache = {}
        self.n = 0
        self.vars = set(var_names)

    def tmp(self, key, rhs):
        if key in self.cache:
            return self.cache[key]
        name = f"t{self.n}"
        self.n += 1
        self.lines.append(f"    const float {name} = {rhs};")
        self.cache[key] = name
        return name

    # value = ('c', python number) | ('v', c-expression-name)
    def visit(self, node):
        if isinstance(node, ast.Constant):
            return ("c", node.value)
        if isinstance(node, ast.Name):
            if node.id == "pi":          # lambdify's namespace binds `pi` to math.pi (a float)
                return ("c", math.pi)
            if node.id not in self.vars:
                raise ValueError(f"unknown symbol {node.id}")
            return ("v", node.id)
        if isinstance(node, ast.UnaryOp):
            k, v = self.visit(node.operand)
            if isinstance(node.op, ast.USub):
                return ("c", -v) if k == "c" else ("v", self.tmp(("neg", v), f"-{v}"))
            if isinstance(node.op, ast.UAdd):
                return (k, v)
            raise ValueError(ast.dump(node))
        if isinstance(node, ast.Call):
            fn = node.func.id
            (k, v), = [self.visit(a) for a in node.args]
            if k == "c":
                return ("c", {"sin": math.sin, "cos": math.cos, "sqrt": math.sqrt}[fn](v))
            cf = {"sin": "sinf", "cos": "cosf", "sqrt": "sqrtf"}[fn]
            return ("v", self.tmp((fn, v), f"{cf}({v})"))
        if isinstance(node, ast.BinOp):
            return self.binop(node.op, self.visit(node.left), self.visit(node.right))
        raise ValueError(ast.dump(node))

    def binop(self, op, a, b):
        (ka, va), (kb, vb) = a, b
        if ka == "c" and kb == "c":
            if isinstance(op, ast.Add):
                return ("c", va + vb)
            if isinstance(op, ast.Sub):
                return ("c", va - vb)
            if isinstance(op, ast.Mult):
                return ("c", va * vb)
            if isinstance(op, ast.Div):
                return ("c", va / vb)
            if isinstance(op, ast.Pow):
                return ("c", va ** vb)
            raise ValueError(op)
        sa = va if ka == "v" else f32_literal(va)
        sb = vb if kb == "v" else f32_literal(vb)
        if isinstance(op, ast.Add):
            x, y = sorted([sa, sb])  # commutative: canonical key
            return ("v", self.tmp(("add", x, y), f"__fadd_rn({sa}, {sb})"))
        if isinstance(op, ast.Mult):
            x, y = sorted([sa, sb])
            return ("v", self.tmp(("mul", x, y), f"__fmul_rn({sa}, {sb})"))
        if isinstance(op, ast.Sub):
            return ("v", self.tmp(("sub", sa, sb), f"__fsub_rn({sa}, {sb})"))
        if isinstance(op, ast.Div):
            if kb == "c":       # tensor / python scalar -> a * (1.0f / b)   [ATen CUDA]
                inv = f32_literal(np.float32(1.0) / np.float32(vb))
                return ("v", self.tmp(("mul", *sorted([sa, inv])), f"__fmul_rn({sa}, {inv})"))
            if ka == "c":       # python scalar / tensor -> reciprocal(b) * a [Tensor.__rtruediv__]
                rcp = self.tmp(("rcp", sb), f"__fdiv_rn(1.0f, {sb})")
                return ("v", self.tmp(("mul", *sorted([rcp, sa])), f"__fmul_rn({rcp}, {sa})"))
            return ("v", self.tmp(("div", sa, sb), f"__fdiv_rn({sa}, {sb})"))
        if isinstance(op, ast.Pow):
            if ka == "v" and kb == "c":
                if vb == 2:
                    return ("v", self.tmp(("mul", sa, sa), f"__fmul_rn({sa}, {sa})"))
                if vb == 3:
                    sq = self.tmp(("mul", sa, sa), f"__fmul_rn({sa}, {sa})")
                    return ("v", self.tmp(("mul", *sorted([sq, sa])), f"__fmul_rn({sq}, {sa})"))
                if vb == 0.5:
                    return ("v", self.tmp(("sqrt", sa), f"sqrtf({sa})"))
                if vb == 1:
                    return ("v", sa)
                return ("v", self.tmp(("pow", sa, sb), f"powf({sa}, {sb})"))
            raise ValueError("only tensor ** python-scalar is supported")
        raise ValueError(op)


def emit_function(name, var_names, sources, doc=""):
    """One __device__ function evaluating all `sources`; results land in out[0..len)."""
    em = _Emitter(var_names)
    results = []
    for src in sources:
        tree = ast.parse(src.strip(), mode="eval").body
        k, v = em.visit(tree)
        results.append(v if k == "v" else f32_literal(v))
    args = ", ".join(f"const float {v}" for v in var_names)
    body = "\n".join(em.lines)
    stores = "\n".join(f"    out[{i}] = {r};" for i, r in enumerate(results))
    n = len(sources)
    return (f"// {doc}\n"
            f"__device__ __forceinline__ void {name}({args}, float (&out)[{n}]) {{\n"
            f"{body}\n{stores}\n}}\n")


def emit_bessel_orders(ns, nr, bessel_sources):
    """bessel() split by order l: bessel_l<l>(x, out[NR]) evaluates entries l*NR .. l*NR+NR-1 with the same expression
    trees (so the same roundings) and bessel_order(l, x, out) dispatches on a block-uniform l -- the edge-basis kernel
    spreads one edge's NS orders over NS threads instead of one thread walking ~80 sinf / cosf calls."""
    parts = []
    for l in range(ns):
        parts.append(emit_function(f"bessel_l{l}", ["x"], bessel_sources[l * nr:(l + 1) * nr],
                                   f"bessel() entries of order l = {l}"))
    cases = "\n".join(f"        case {l}: bessel_l{l}(x, out); break;" for l in range(ns))
    parts.append("// order l of bessel(); l must be uniform over the warp\n"
                 f"__device__ __forceinline__ void bessel_order(const int l, const float x, float (&out)[{nr}]) {{\n"
                 f"    switch (l) {{\n{cases}\n        default: break;\n    }}\n}}\n")
    return "\n".join(parts)


def emit_header(tag, flavor, num_spherical, num_radial, sources):
    """Full generated header for one (flavor, ns, nr)."""
    ns, nr = num_spherical, num_radial
    parts = [
        "// GENERATED by dig_b200/codegen.py -- do not edit.\n"
        f"// flavor={flavor} num_spherical={ns} num_radial={nr}\n"
        "// One correctly-rounded fp32 op per Python arithmetic node of the reference's\n"
        "// lambdified closed forms (SURVEY.md 5.9c); see dig_b200/basis.py for provenance.\n"
        "#pragma once\n",
        f"namespace basis_{tag} {{\n",
        f"constexpr int NS = {ns};\nconstexpr int NR = {nr};\n"
        f"constexpr int N_BESSEL = {len(sources['bessel'])};\n"
        f"constexpr int N_YL0 = {len(sources['yl0'])};\n"
        f"constexpr int N_YLM = {len(sources['ylm'])};\n",
        emit_function("bessel", ["x"], sources["bessel"],
                      "normalised spherical Bessel j_l(z_ln x); index l*NR + n"),
        emit_bessel_orders(ns, nr, sources["bessel"]),
        emit_function("yl0", ["theta"], sources["yl0"], "real spherical harmonics Y_l^0(theta)"),
        emit_function("ylm", ["theta", "phi"], sources["ylm"],
                      "real spherical harmonics, reference flat order"),
        emit_function("bessel_dx", ["x"], sources["bessel_dx"],
                      "d/dx of bessel() (symbolic derivative of the same closed forms; force path)"),
        emit_function("yl0_dtheta", ["theta"], sources["yl0_dtheta"], "d/dtheta of yl0() (force path)"),
        emit_function("ylm_dtheta", ["theta", "phi"], sources["ylm_dtheta"], "d/dtheta of ylm() (force path)"),
        emit_function("ylm_dphi", ["theta", "phi"], sources["ylm_dphi"], "d/dphi of ylm() (force path)"),
        "}  // namespace\n",
    ]
    return "\n".join(parts)


def emit_header_second_order(tag, flavor, num_spherical, num_radial, sources):
    """Header of the second derivatives (basis.basis_sources_second_order) for one (flavor, ns, nr): the reverse mode of
    the tangent kernels (Hessian-vector products) is their only reader, so they stay out of the first-order header."""
    ns, nr = num_spherical, num_radial
    parts = [
        "// GENERATED by dig_b200/codegen.py -- do not edit.\n"
        f"// flavor={flavor} num_spherical={ns} num_radial={nr}: second derivatives of the closed forms of\n"
        f"// basis_{tag}.cuh (symbolic, same fp32 rounding rules); see dig_b200/basis.py.\n"
        "#pragma once\n",
        f"namespace basis_{tag} {{\n",
        emit_function("bessel_dxx", ["x"], sources["bessel_dxx"], "d2/dx2 of bessel()"),
        emit_function("yl0_dtheta2", ["theta"], sources["yl0_dtheta2"], "d2/dtheta2 of yl0()"),
        emit_function("ylm_dtheta2", ["theta", "phi"], sources["ylm_dtheta2"], "d2/dtheta2 of ylm()"),
        emit_function("ylm_dtheta_dphi", ["theta", "phi"], sources["ylm_dtheta_dphi"], "d2/dtheta dphi of ylm()"),
        emit_function("ylm_dphi2", ["theta", "phi"], sources["ylm_dphi2"], "d2/dphi2 of ylm()"),
        "}  // namespace\n",
    ]
    return "\n".join(parts)


CONFIGS = {
    # tag: (flavor, num_spherical, num_radial)
    "dimenet_7_6": ("dimenet", 7, 6),      # SphereNet / DimeNet++ defaults
    "dimenet_3_6": ("dimenet", 3, 6),      # SphereNet notebook example (ns=3)
    "gemnet_2_3": ("gemnet", 2, 3),        # ComENet defaults
    "gemnet_2_6": ("gemnet", 2, 6),        # ProNet defaults (pronet/features.py is comenet/features.py with nr = 6)
}
# configurations with a second-order header (DimeNet++ / SphereNet / ComENet Hessians)
SECOND_ORDER = ("dimenet_7_6", "dimenet_3_6", "gemnet_2_3")


def generate_all(out_dir, force=False):
    import os
    from . import basis
    os.makedirs(out_dir, exist_ok=True)
    written = []
    for tag, (flavor, ns, nr) in CONFIGS.items():
        path = os.path.join(out_dir, f"basis_{tag}.cuh")
        if os.path.exists(path) and not force:
            continue
        src = basis.basis_sources(flavor, ns, nr)
        with open(path, "w") as fh:
            fh.write(emit_header(tag, flavor, ns, nr, src))
        written.append(path)
    for tag in SECOND_ORDER:
        flavor, ns, nr = CONFIGS[tag]
        path = os.path.join(out_dir, f"basis_{tag}_d2.cuh")
        if os.path.exists(path) and not force:
            continue
        with open(path, "w") as fh:
            fh.write(emit_header_second_order(tag, flavor, ns, nr, basis.basis_sources_second_order(flavor, ns, nr)))
        written.append(path)
    return written


if __name__ == "__main__":
    import os
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    print(generate_all(os.path.join(here, "csrc", "generated"), force="--force" in sys.argv))
