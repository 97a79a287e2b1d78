"""GPU tests of the argument rules every entry point that takes resident polynomials applies, before it launches anything:

- an unknown handle, or another lane's, is "unknown polynomial handle";
- a shared output is "the polynomial is shared (read-only)"; shared inputs are allowed;
- every polynomial is of one field ("the polynomials live in different fields"; the MSM-side calls want the curve's scalar
  field) and holds the range the call needs ("a polynomial holds fewer than <len> elements"), a range whose end would wrap
  included;
- a failure on an element of a handle array names it: "<who>: <name>[i]: <reason>";
- where outputs may not alias, "<a> is also <b>", the output first ("dst[1] is also dst[0]", "dst is also src").

For every row of the table the call fails, its message starts with the entry point's name, the argument and the reason, no
kernel is launched, and no polynomial changes.  Each entry point's call with the default handles succeeds, so every row
fails for the one argument it replaces."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref  # noqa: E402
from tests.test_gpu_lanes import _bind, _create, _destroy, _err, _lib  # noqa: E402

SEED = 0x41524753
K, N = 6, 1 << 6
UNKNOWN = 0xDEADBEEF
WRAP = (1 << 64) - 2                                                   # SIZE_MAX - 1: off + 4 wraps to 2
MIXED = "the polynomials live in different fields"


def _fe_np(x):
    from halo2_b200 import lib as L
    return L.fe_bytes(x)


def _fe(x=3):
    return _fe_np(x).ctypes.data_as(ctypes.c_void_p)


def _arr(hs):
    return (ctypes.c_uint64 * len(hs))(*hs)


def _u64(h):
    return ctypes.c_uint64(h)


def _sz(n):
    return ctypes.c_size_t(n)


def _u32(n):
    return ctypes.c_uint32(n)


class Spec:
    """One entry point: call(outs, ins) with handle lists, in the order the library looks them up.  `onames` / `inames` name
    each slot as the messages do: "dst" for a single handle, "dst[0]" for an element of an array.  `alias`: the call has the
    aliasing rule; `field`: the reason a polynomial of the other field gives (None: one polynomial, no rule); `short`:
    whether a 4-element polynomial is too short in every slot; `extra`: more rows (label, call(outs, ins), message after
    "<prefix>: ")."""

    def __init__(self, name, outs, onames, ins, inames, call, alias=False, field=MIXED, short=True,
                 prefix=None, extra=()):
        assert len(outs) == len(onames) and len(ins) == len(inames)
        self.name, self.outs, self.onames, self.ins, self.inames, self.call = name, outs, onames, ins, inames, call
        self.alias, self.field, self.short, self.extra = alias, field, short, extra
        self.prefix = prefix or name


def _specs(prm):
    lib = _lib()
    zeros = np.zeros((N, 32), dtype=np.uint8)
    down = np.zeros((N, 32), dtype=np.uint8)
    pts = np.ascontiguousarray(np.stack([_fe_np(5), _fe_np(7)]))
    res = np.zeros(4 * 96, dtype=np.uint8)
    u = np.ascontiguousarray(np.stack([_fe_np(j + 2) for j in range(K)]))
    t = np.ascontiguousarray(np.stack([_fe_np(9)]))
    blind = np.ascontiguousarray(np.stack([_fe_np(j + 11) for j in range(4)]))
    vals = np.ascontiguousarray(np.stack([_fe_np(j + 21) for j in range(8)]))
    code = np.array([[0, 0, 0, 0]], dtype=np.uint32)                  # POLY 0
    ident = np.stack(np.meshgrid(np.arange(2), np.arange(N), indexing="ij"), axis=-1).astype(np.uint32)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    sess = ctypes.c_uint64(0)

    def ipa(o, i):
        rc = lib.h2_ipa_begin_poly(prm._h_g, _u32(K), _u64(i[0]), _fe(), 0, ctypes.byref(sess))
        if rc == 0:                                                     # the default call opens a session: abort it
            assert lib.h2_ipa_finish(sess, 0, None) == 0, _err()
        return rc

    copy = lambda do=0, so=0: lambda o, i: lib.h2_poly_copy(_u64(o[0]), _sz(do), _u64(i[0]), _sz(so), _sz(4 if do or so else N))
    set_rows = lambda start=N - 2: lambda o, i: lib.h2_poly_set_rows(_arr(o), _sz(2), _sz(start), _sz(2 if start == N - 2 else 4), vp(vals), 0)
    return [
        Spec("h2_poly_upload", ["e"], ["poly"], [], [], lambda o, i: lib.h2_poly_upload(_u64(o[0]), vp(zeros), _sz(N), 0), field=None),
        Spec("h2_poly_download", [], [], ["a"], ["poly"], lambda o, i: lib.h2_poly_download(_u64(i[0]), vp(down), _sz(N), 0), field=None),
        Spec("h2_poly_add_at", ["e"], ["poly"], [], [], lambda o, i: lib.h2_poly_add_at(_u64(o[0]), _sz(1), _fe(), 0), field=None, short=False),
        Spec("h2_poly_copy", ["e"], ["dst"], ["a"], ["src"], copy(),
             extra=[("dst-wrap", copy(do=WRAP), "a polynomial holds fewer than dst_off + len elements"),
                    ("src-wrap", copy(so=WRAP), "a polynomial holds fewer than src_off + len elements")]),
        Spec("h2_poly_lagrange_to_coeff", ["e"], ["dst"], ["a"], ["src"],
             lambda o, i: lib.h2_poly_lagrange_to_coeff(_u64(o[0]), _u64(i[0]), _u32(K), _fe(), _fe(), 0)),
        Spec("h2_poly_coeff_to_extended", ["e"], ["dst"], ["a"], ["src"],
             lambda o, i: lib.h2_poly_coeff_to_extended(_u64(o[0]), _u64(i[0]), _u32(K - 1), _u32(K), _fe(), _fe(), 0)),
        Spec("h2_poly_extended_to_coeff", ["e"], ["dst"], ["a"], ["src"],
             lambda o, i: lib.h2_poly_extended_to_coeff(_u64(o[0]), _u64(i[0]), _u32(K), _fe(), _fe(), _fe(), _sz(N), 0)),
        Spec("h2_poly_lagrange_to_coeff_batch", ["e", "f"], ["dst[0]", "dst[1]"], ["a", "b"], ["src[0]", "src[1]"],
             lambda o, i: lib.h2_poly_lagrange_to_coeff_batch(_arr(o), _arr(i), _sz(2), _u32(K), _fe(), _fe(), 0), alias=True),
        Spec("h2_poly_coeff_to_extended_batch", ["e", "f"], ["dst[0]", "dst[1]"], ["a", "b"], ["src[0]", "src[1]"],
             lambda o, i: lib.h2_poly_coeff_to_extended_batch(_arr(o), _arr(i), _sz(2), _u32(K - 1), _u32(K), _fe(), _fe(), 0), alias=True),
        Spec("h2_poly_set_rows", ["e", "f"], ["polys[0]", "polys[1]"], [], [], set_rows(), alias=True,
             extra=[("wrap", set_rows(start=WRAP), "polys[0]: a polynomial holds fewer than start + rows elements")]),
        Spec("h2_poly_eval", [], [], ["a", "b"], ["polys[0]", "polys[1]"], lambda o, i: lib.h2_poly_eval(_arr(i), _sz(2), _sz(N), vp(pts), 0, vp(res))),
        Spec("h2_poly_inner_product", [], [], ["a", "b", "c", "d"], ["a[0]", "a[1]", "b[0]", "b[1]"],
             lambda o, i: lib.h2_poly_inner_product(_arr(i[:2]), _arr(i[2:]), _sz(2), _sz(N), 0, vp(res))),
        Spec("h2_poly_kate_division", ["e", "f"], ["dst[0]", "dst[1]"], ["a", "b"], ["src[0]", "src[1]"],
             lambda o, i: lib.h2_poly_kate_division(_arr(o), _arr(i), _sz(2), _sz(N), vp(pts), 0), alias=True),
        Spec("h2_poly_divide_by_vanishing", ["e"], ["poly"], [], [], lambda o, i: lib.h2_poly_divide_by_vanishing(_u64(o[0]), _u32(K), vp(t), _u32(1), 0),
             field=None),
        Spec("h2_poly_eval_ast", ["e"], ["out"], ["a", "b"], ["polys[0]", "polys[1]"],
             lambda o, i: lib.h2_poly_eval_ast(_u64(o[0]), _arr(i), _sz(len(i)), _u32(K), vp(code), _sz(1), None, _sz(0), None, None, 0),
             alias=True),
        Spec("h2_poly_batch_invert", ["e"], ["poly"], [], [], lambda o, i: lib.h2_poly_batch_invert(_u64(o[0]), _sz(N)), field=None),
        Spec("h2_poly_running_product", ["e"], ["dst"], ["a"], ["src"],
             lambda o, i: lib.h2_poly_running_product(_u64(o[0]), _u64(i[0]), _sz(N), _fe(), 0), alias=True),
        Spec("h2_poly_lookup_permute", ["e", "f"], ["out_input", "out_table"], ["a", "a"], ["input", "table"],
             lambda o, i: lib.h2_poly_lookup_permute(_u64(i[0]), _u64(i[1]), _sz(N - 2), _u64(o[0]), _u64(o[1])), alias=True),
        Spec("h2_poly_lookup_permuted", ["e", "f"], ["out_inputs[0]", "out_tables[0]"], ["a", "a"], ["inputs[0]", "tables[0]"],
             lambda o, i: lib.h2_poly_lookup_permuted(_arr(o[:1]), _arr(o[1:]), _sz(1), _arr(i[:1]), _arr(i[1:]), _u32(K), vp(blind), _u32(1), 0),
             alias=True),
        Spec("h2_poly_compute_s", ["e"], ["dst"], [], [], lambda o, i: lib.h2_poly_compute_s(_u64(o[0]), vp(u), _u32(K), _fe(), 0, 0), field=None),
        Spec("h2_poly_scale_add", ["e"], ["dst"], ["a"], ["src"], lambda o, i: lib.h2_poly_scale_add(_u64(o[0]), _fe(2), _u64(i[0]), _fe(3), _sz(N), 0),
             alias=True),
        Spec("h2_poly_permutation_sigma", ["e", "f"], ["dst[0]", "dst[1]"], [], [],
             lambda o, i: lib.h2_poly_permutation_sigma(_arr(o), _sz(2), _u32(K), vp(ident), _fe(), _fe(), 0), alias=True),
        Spec("h2_poly_permutation_sigma_copies", ["e", "f"], ["dst[0]", "dst[1]"], [], [],
             lambda o, i: lib.h2_poly_permutation_sigma_copies(_arr(o), _sz(2), _u32(K), None, _sz(0), _fe(), _fe(), 0), alias=True),
        Spec("h2_poly_permutation_product", ["e", "f"], ["z_out[0]", "z_out[1]"], ["a", "b", "c", "d"],     # one proof, 2 columns in sets of 1
             ["columns[0]", "columns[1]", "sigmas[0]", "sigmas[1]"],
             lambda o, i: lib.h2_poly_permutation_product(_arr(o), _sz(1), _arr(i[:2]), _arr(i[2:]), _sz(2), _u32(1), _u32(K), _fe(), _fe(), _fe(),
                                                          _fe(), None, _u32(0), 0), alias=True),
        Spec("h2_poly_lookup_product", ["e", "f"], ["z_out[0]", "z_out[1]"], ["a", "b", "c", "d", "a", "b", "c", "d"],
             [f"{n}[{j}]" for n in ("inputs", "tables", "permuted_inputs", "permuted_tables") for j in range(2)],
             lambda o, i: lib.h2_poly_lookup_product(_arr(o), _sz(2), _arr(i[0:2]), _arr(i[2:4]), _arr(i[4:6]), _arr(i[6:8]), _u32(K), _fe(), _fe(),
                                                     None, _u32(0), 0), alias=True),
        Spec("h2_msm_registered_polys", [], [], ["a", "b"], ["polys[0]", "polys[1]"],
             lambda o, i: lib.h2_msm_registered_polys(prm._h_g, _arr(i), _sz(2), _sz(N), None, 0, vp(res)),
             field="the polynomial is not over the curve's scalar field"),
        Spec("h2_msm_registered_polys_affine", [], [], ["a", "b"], ["polys[0]", "polys[1]"],
             lambda o, i: lib.h2_msm_registered_polys_affine(prm._h_g, _arr(i), _sz(2), _sz(N), None, 0, vp(res)),
             field="the polynomial is not over the curve's scalar field", prefix="h2_msm_registered_polys"),
        Spec("h2_ipa_begin_poly", [], [], ["a"], ["p_prime_poly"], ipa, field="the polynomial is not over the curve's scalar field"),
    ]


def _rows(spec, P):
    """(label, outs, ins, message after "<prefix>: ", call) for every rejection that applies to `spec`, as handles."""
    h = lambda names: [P[n] if isinstance(n, str) else n for n in names]
    names = spec.onames + spec.inames                                  # every slot, in lookup order
    at = lambda slot, reason: f"{slot}: {reason}" if "[" in slot else reason
    bad = [("unknown", UNKNOWN, "unknown polynomial handle"), ("foreign", "foreign", "unknown polynomial handle")]
    if spec.field:
        bad.append(("field", "fq", spec.field))
    if spec.short:
        bad.append(("short", "short", "a polynomial holds fewer than"))
    for j in range(len(names)):
        for label, v, reason in bad + ([("shared", "shared", "the polynomial is shared (read-only)")] if j < len(spec.outs) else []):
            slots = spec.outs + spec.ins
            slots[j] = v
            # without a given field it is the first polynomial's: one of the other field in the first slot fails the second
            slot = names[1] if label == "field" and spec.field == MIXED and j == 0 else names[j]
            yield f"{names[j]}-{label}", h(slots[:len(spec.outs)]), h(slots[len(spec.outs):]), at(slot, reason), spec.call
    if spec.alias:
        if len(spec.outs) > 1:
            yield "out-twice", h([spec.outs[0], spec.outs[0]] + spec.outs[2:]), h(spec.ins), f"{spec.onames[1]} is also {spec.onames[0]}", spec.call
        if spec.ins:
            other = spec.inames[spec.ins.index(spec.ins[-1])]
            yield "out-is-input", h([spec.ins[-1]] + spec.outs[1:]), h(spec.ins), f"{spec.onames[0]} is also {other}", spec.call
    for label, call, msg in spec.extra:
        yield label, h(spec.outs), h(spec.ins), msg, call


@pytest.fixture(scope="module")
def env():
    import halo2_b200 as eng
    from halo2_b200 import lib as L
    L.init()
    lane = _create()
    assert _bind(lane) == 0
    foreign = eng.ResidentPoly("fp", N, cref.gen_scalars("fp", SEED, N))
    assert _bind(0) == 0
    P = {n: eng.ResidentPoly("fp", N, cref.gen_scalars("fp", SEED + j + 1, N)) for j, n in enumerate("abcdef")}
    P["fq"] = eng.ResidentPoly("fq", N, cref.gen_scalars("fq", SEED + 7, N))
    P["short"] = eng.ResidentPoly("fp", 4, cref.gen_scalars("fp", SEED + 8, 4))
    P["shared"] = eng.ResidentPoly("fp", N, cref.gen_scalars("fp", SEED + 9, N)).share()
    pts = cref.gen_points("vesta", SEED, N + 2)
    prm = eng.Params("vesta", K, pts[:N], eng.lagrange_generators("vesta", K, pts[:N]), pts[N:N + 1], u=pts[N + 1:])
    try:
        yield P, {**{n: p._h.value for n, p in P.items()}, "foreign": foreign._h.value}, prm
    finally:
        prm.close()
        for p in P.values():
            p.close()
        _bind(lane)
        foreign.close()
        _bind(0)
        _destroy(lane)


def test_defaults_succeed(env):
    P, H, prm = env
    for spec in _specs(prm):
        assert spec.call([H[n] for n in spec.outs], [H[n] for n in spec.ins]) == 0, (spec.name, _err())
    # with the default handles, in-place columns of the batch transforms are allowed
    lib = _lib()
    assert lib.h2_poly_lagrange_to_coeff_batch(_arr([H["e"], H["f"]]), _arr([H["e"], H["f"]]), _sz(2), _u32(K), _fe(), _fe(), 0) == 0, _err()


def test_rejections_name_the_argument(env):
    P, H, prm = env
    lib = _lib()
    specs = _specs(prm)
    assert len(specs) == 28
    rows, wrong = 0, []
    for spec in specs:
        for label, outs, ins, reason, call in _rows(spec, H):
            before = {n: p.download().tobytes() for n, p in P.items()}
            launches = lib.h2_launch_count()
            rc = call(outs, ins)
            msg = _err() if rc else ""
            launched = lib.h2_launch_count() - launches
            changed = [n for n, p in P.items() if p.download().tobytes() != before[n]]
            if rc == 0 or not msg.startswith(f"{spec.prefix}: {reason}") or launched or changed:
                wrong.append(f"{spec.name} {label}: rc {rc}, {launched} launches, changed {changed}: {msg!r}")
            rows += 1
    assert rows == 344
    assert not wrong, "\n".join(wrong)
