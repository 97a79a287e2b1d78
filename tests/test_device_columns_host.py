"""CPU checks of the device-memory column transfers (h2_poly_upload_dev / h2_poly_download_dev, K25 columns_io.cuh): the
kernel body on the host emulation against the field's Montgomery conversion and the host path's, and the Python layer's
refusals over the ABI stand-in."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import cref, pasta
from tests.fake_device_columns import installed
from tests.kernel_emul import build as emul_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 1 << 256
LENS = (0, 1, 127, 128, 129, 1 << 12)


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def _ints(a):
    return [int.from_bytes(r.tobytes(), "little") for r in a]


def _inputs(field, n, seed):
    """n 256-bit elements: random ones, and values >= p, all-ones bytes and the edges around p among them."""
    m = pasta.FIELDS[field]
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    special = [0, 1, m - 1, m, m + 1, 2 * m, 3 * m, R - 1, R - 2]
    for i, x in enumerate(special[:n]):
        a[(i * 37) % n] = np.frombuffer(x.to_bytes(32, "little"), dtype=np.uint8)
    return a


def _io(emu, field, to_dev, canon, res, caller):
    count = len(res)
    emu.emu_columns_io(cref.FIELD_ID[field], to_dev, canon, ctypes.c_uint64(count), (ctypes.c_void_p * count)(*[r.ctypes.data for r in res]),
                       (ctypes.c_void_p * count)(*[c.ctypes.data for c in caller]), (ctypes.c_uint64 * count)(*[c.shape[0] for c in caller]))


def _host_path(emu, field, to_mont, a):
    """What h2_poly_upload / h2_poly_download's conversion (convert_field) makes of the elements."""
    b = np.ascontiguousarray(a).copy()
    emu.emu_convert(cref.FIELD_ID[field], to_mont, ctypes.c_uint64(b.shape[0]), cref._p(b))
    return b


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("repr_", ["canonical", "montgomery"])
def test_emul_columns_io(emu, field, repr_):
    """Every length of LENS as one column of one call, in both directions.  Import: x R mod p for x < p, the host path's
    bytes for every input (>= p included, no range check); Montgomery input is copied.  Export: x R^-1 mod p for every
    input.  Elements past a column's length are left alone."""
    m, canon = pasta.FIELDS[field], int(repr_ == "canonical")
    rinv = pow(R, -1, m)
    src = [_inputs(field, max(n, 1), 7 + n)[:n] for n in LENS]
    fill = np.uint8(0xA5)
    res = [np.full((n + 3, 32), fill, dtype=np.uint8) for n in LENS]
    _io(emu, field, 1, canon, res, src)
    for n, s, r in zip(LENS, src, res):
        assert (r[n:] == fill).all(), n
        if not canon:
            assert (r[:n] == s).all(), n
            continue
        assert (r[:n] == _host_path(emu, field, 1, s)).all(), n
        for x, y in zip(_ints(s), _ints(r[:n])):
            if x < m:
                assert y == x * R % m, (n, hex(x))
    out = [np.full((n + 3, 32), fill, dtype=np.uint8) for n in LENS]
    views = [o[:n] for o, n in zip(out, LENS)]
    _io(emu, field, 0, canon, [np.ascontiguousarray(s) for s in src], views)
    for n, s, o in zip(LENS, src, out):
        assert (o[n:] == fill).all(), n
        want = s if not canon else cref.ints_to_bytes([x * rinv % m for x in _ints(s)]).reshape(-1, 32)
        assert (o[:n] == want[:n]).all(), n
        if canon:
            assert (o[:n] == _host_path(emu, field, 0, s)).all(), n


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_columns_io_round_trip(emu, field):
    """Canonical values go up and come back unchanged, several columns of different lengths per call."""
    lens = (5, 300, 1, 257)
    vals = [cref.gen_scalars(field, 40 + i, n) for i, n in enumerate(lens)]
    res = [np.zeros((n, 32), dtype=np.uint8) for n in lens]
    _io(emu, field, 1, 1, res, vals)
    back = [np.zeros((n, 32), dtype=np.uint8) for n in lens]
    _io(emu, field, 0, 1, res, back)
    for v, b in zip(vals, back):
        assert (v == b).all()


# ---- the Python layer over the ABI stand-in ----

def _dev_calls(fake):
    return [c for c in fake.calls if c.endswith("_dev")]


def test_tensor_refusals_before_any_call():
    torch = pytest.importorskip("torch")
    from halo2_b200 import poly
    with installed() as fake:
        p = poly.ResidentPoly("fp", 8)
        good = torch.zeros((8, 32), dtype=torch.uint8)
        cases = [
            (np.zeros((8, 32), dtype=np.uint8), TypeError, "expected a torch.Tensor"),
            (good.to(torch.int32), ValueError, "dtype"),
            (torch.zeros((8, 31), dtype=torch.uint8), ValueError, "shape"),
            (torch.zeros(8 * 32, dtype=torch.uint8), ValueError, "shape"),
            (torch.zeros((32, 8), dtype=torch.uint8).t(), ValueError, "not contiguous"),
            (torch.zeros((16, 32), dtype=torch.uint8)[::2], ValueError, "not contiguous"),
            (torch.zeros((9, 32), dtype=torch.uint8), ValueError, "9 rows, the polynomial holds 8"),
            (good, ValueError, "a CPU tensor"),
        ]
        for t, exc, msg in cases:
            with pytest.raises(exc, match=msg):
                p.upload_tensor(t)
            with pytest.raises(exc, match=msg):
                poly.upload_tensors_resident([p], [t])
        with pytest.raises(ValueError, match="a CPU tensor"):
            poly.ResidentPoly.from_tensor("fp", good)
        with pytest.raises(ValueError, match="a CPU tensor"):
            p.to_tensor(out=good)
        with pytest.raises(ValueError, match="repr"):
            p.upload_tensor(good, repr="mont")
        with pytest.raises(ValueError, match="lengths\\[0\\] = 9"):
            p.to_tensor(length=9)
        with pytest.raises(ValueError, match="one tensor per polynomial"):
            poly.upload_tensors_resident([p], [])
        assert _dev_calls(fake) == []


def test_pointer_helper_over_the_stand_in():
    """The pointer-level helper with host buffers standing for device memory: one call for several columns, the same
    values as the host upload, both reprs; the library's refusals before any launch."""
    from halo2_b200 import lib as L, poly
    m = pasta.FIELDS["fq"]
    with installed() as fake:
        lens = [3, 0, 17]
        vals = [cref.gen_scalars("fq", 90 + i, n) if n else np.zeros((0, 32), np.uint8) for i, n in enumerate(lens)]
        ps = [poly.ResidentPoly("fq", 20) for _ in lens]
        poly.upload_dev_resident(ps, [v.ctypes.data if v.size else 0 for v in vals], lens, L.REPR_CANONICAL, 0)
        assert _dev_calls(fake) == ["h2_poly_upload_dev"]
        for p, v, n in zip(ps, vals, lens):
            assert (p.download(n) == v).all()
            assert not p.download()[n:].any()
        mont = np.ascontiguousarray(cref.ints_to_bytes([x * R % m for x in _ints(vals[2])]).reshape(-1, 32))
        q = poly.ResidentPoly("fq", 17)
        poly.upload_dev_resident([q], [mont.ctypes.data], [17], L.REPR_MONTGOMERY, 0)
        assert (q.download() == vals[2]).all()
        outs = [np.zeros((n, 32), np.uint8) for n in (3, 17)]
        poly.download_dev_resident([ps[0], q], [o.ctypes.data for o in outs], [3, 17], L.REPR_CANONICAL, 0)
        assert (outs[0] == vals[0]).all() and (outs[1] == vals[2]).all()
        poly.download_dev_resident([q], [outs[1].ctypes.data], [17], L.REPR_MONTGOMERY, 0)
        assert (outs[1] == mont).all()

        before = list(fake.calls)
        buf = np.zeros((40, 32), np.uint8)
        other = poly.ResidentPoly("fp", 20)
        shared = poly.ResidentPoly("fq", 20).share()
        refusals = [
            (poly.upload_dev_resident, [ps[0]], [buf.ctypes.data], [21], "polys\\[0\\]: a polynomial holds fewer than lens\\[0\\] elements"),
            (poly.upload_dev_resident, [ps[0], ps[0]], [buf.ctypes.data] * 2, [1, 1], "polys\\[1\\] is also polys\\[0\\]"),
            (poly.upload_dev_resident, [shared], [buf.ctypes.data], [1], "shared"),
            (poly.upload_dev_resident, [ps[0], other], [buf.ctypes.data] * 2, [1, 1], "different fields"),
            (poly.upload_dev_resident, [ps[0]], [buf.ctypes.data + 8], [2], "d_src\\[0\\]: not 16-byte aligned"),
            (poly.upload_dev_resident, [ps[0]], [0], [2], "d_src\\[0\\]: null pointer"),
            (poly.download_dev_resident, [ps[0], ps[2]], [buf.ctypes.data, buf.ctypes.data + 64], [3, 3], "d_dst\\[1\\]: overlaps d_dst\\[0\\]"),
        ]
        for fn, hs, ptrs, ls, msg in refusals:
            with pytest.raises(L.H2Error, match=msg):
                fn(hs, ptrs, ls, L.REPR_CANONICAL, 0)
        assert fake.calls == before and not buf.any()
        # a shared polynomial is read by the download; a shared source of one call may repeat
        poly.download_dev_resident([shared, shared], [buf.ctypes.data, buf.ctypes.data + 64], [2, 2], L.REPR_CANONICAL, 0)


def test_import_without_torch():
    """The package, its phases and is_device_tensor work where torch cannot be imported."""
    code = ("import sys; sys.modules['torch'] = None\n"
            "import numpy as np, halo2_b200\n"
            "from halo2_b200 import poly, columns, keygen\n"
            "assert not poly.is_device_tensor(np.zeros((2, 32), np.uint8)) and not poly.is_device_tensor([1, 2])\n"
            "assert sys.modules['torch'] is None\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
