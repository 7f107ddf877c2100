"""The grouped weight-gradient kernel (wgrad_group.cuh) on its own, through dwbc_debug_wgrad_group, against float64.

Every operand storage is NaN wherever the kernel must not look: rows past R of a tile image (the image holds whole 128-row tiles), the
padding columns of a row-major row, the storage rows a gather index skips.  The kernel stages whole 16-byte pieces and whole image
blocks, so it reads such values and must mask them.  Operands are tile images (128 wide), row-major with 16-byte aligned rows (16-byte
copies), row-major with unaligned rows (plain loads) and rows gathered through an index."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = [1, 6, 12, 20, 24, 64, 76, 100, 128]
TOL = {1: 2e-5, 0: 3e-3}          # ||dW - ref|| / || |G|^T |X| ||: 3xTF32 (fp32-grade), TF32
DB_TOL = 1e-5                     # the bias sums run on the CUDA cores in fp32


class Gemm(C.Structure):
    _fields_ = [("g", C.c_void_p), ("g_idx", C.c_void_p), ("g_image", C.c_int64), ("g_ld", C.c_int64),
                ("x", C.c_void_p), ("x_idx", C.c_void_p), ("x_image", C.c_int64), ("x_ld", C.c_int64),
                ("dw", C.c_void_p), ("lddw", C.c_int64), ("db", C.c_void_p), ("mo", C.c_int64), ("ni", C.c_int64)]


def _image(m):
    """[R, 128] -> tile images, element (r, k) of tile r // 128 at ((r % 128 / 8) * 32 + k / 4) * 32 + (r % 8) * 4 + k % 4; rows past R NaN"""
    r = m.shape[0]
    t = (r + 127) // 128
    pad = torch.full((t * 128, 128), float("nan"), device=m.device)
    pad[:r] = m
    return pad.view(t, 16, 8, 32, 4).permute(0, 1, 3, 2, 4).contiguous().view(-1)


def _operand(kind, rows, ncol, gen, keep):
    """(values [rows, ncol] float32, pointer, idx pointer, image flag, ld); `keep` holds the storages alive"""
    v = torch.randn(rows, ncol, generator=gen, device="cuda")
    if kind == "image":
        assert ncol == 128
        st = _image(v)
        keep.append(st)
        return v, st.data_ptr(), None, 1, 128
    if kind == "row":                      # rows of align_up(ncol, 4) floats: 16-byte copies, padding columns NaN
        ld = (ncol + 3) // 4 * 4
        st = torch.full((rows, ld), float("nan"), device="cuda")
        st[:, :ncol] = v
        keep.append(st)
        return v, st.data_ptr(), None, 0, ld
    if kind == "unaligned":                # rows of ncol + 1 floats from an odd float offset: plain loads
        ld = ncol + 1
        st = torch.full((rows * ld + 1,), float("nan"), device="cuda")
        st[1:].view(rows, ld)[:, :ncol] = v
        keep.append(st)
        return v, st.data_ptr() + 4, None, 0, ld
    assert kind == "gather"                # rows idx[r] of a wider storage (stride 860), columns from float 76 on
    s_rows, stride, off = rows + 37, 860, 76
    st = torch.full((s_rows, stride), float("nan"), device="cuda")
    idx = torch.randperm(s_rows, generator=gen, device="cuda")[:rows].contiguous()
    st[idx, off:off + ncol] = v
    keep += [st, idx]
    return v, st.data_ptr() + 4 * off, idx.data_ptr(), 0, stride


def _kinds(width):
    return ["image", "row", "gather"] if width == 128 else ["row", "unaligned", "gather"]


def _spec(n, seed):
    """n GEMMs with mixed widths and operand kinds"""
    out = []
    for i in range(n):
        mo, ni = WIDTHS[(i + seed) % len(WIDTHS)], WIDTHS[(3 * i + 1 + seed) % len(WIDTHS)]
        out.append((mo, ni, _kinds(mo)[i % 3], _kinds(ni)[(i + 1) % 3], i % 4 != 3))
    return out


def _run(spec, rows, x3, seed=0):
    from dwbc_b200 import _lib as L
    lib = L.lib()
    lib.dwbc_debug_wgrad_group.argtypes = [C.POINTER(Gemm), C.c_int, C.c_int, C.c_int, C.c_void_p]
    gen = torch.Generator(device="cuda").manual_seed(seed)
    keep, descs, refs = [], (Gemm * len(spec))(), []
    for i, (mo, ni, gk, xk, bias) in enumerate(spec):
        g, gp, gi, gim, gld = _operand(gk, rows, mo, gen, keep)
        x, xp, xi, xim, xld = _operand(xk, rows, ni, gen, keep)
        lddw = ni + 3                                           # odd row stride: the scalar atomics of the epilogue
        dw = torch.randn(mo, lddw, generator=gen, device="cuda")
        db = torch.randn(mo, generator=gen, device="cuda") if bias else None
        keep += [dw, db]
        descs[i] = Gemm(gp, gi, gim, gld, xp, xi, xim, xld, dw.data_ptr(), lddw, db.data_ptr() if bias else None, mo, ni)
        g64, x64 = g.double(), x.double()
        refs.append((dw, dw[:, :ni].double() + g64.T @ x64, g64.abs().T @ x64.abs(), db,
                     None if db is None else db.double() + g64.sum(0), g64.abs().sum(0)))
    torch.cuda.synchronize()
    assert lib.dwbc_debug_wgrad_group(descs, len(spec), rows, int(x3), None) == 0
    torch.cuda.synchronize()
    for (dw, ref, scale, db, dbref, dbscale), (mo, ni, gk, xk, _) in zip(refs, spec):
        what = (mo, ni, gk, xk, rows, x3)
        assert torch.isfinite(dw).all(), what
        err = float((dw[:, :ni].double() - ref).norm()) / float(scale.norm())
        assert err <= TOL[int(x3)], (what, err)
        if db is not None:
            assert float((db.double() - dbref).norm()) <= DB_TOL * float(dbscale.norm()), what


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("rows", [1, 63, 64, 129])
def test_one_narrow_gemm_fewer_items_than_sms(rows, x3):
    _run([(1, 1, "row", "row", True)], rows, x3)
    _run([(6, 76, "unaligned", "gather", True)], rows, x3, seed=1)


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("rows", [1, 129, 40960])
def test_two_gemms_image_operands(rows, x3):
    _run([(128, 100, "image", "gather", True), (6, 128, "unaligned", "image", False)], rows, x3)


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("n,rows", [(17, 40960), (17, 132 * 128 + 77), (20, 132 * 128 + 77), (20, 333)])
def test_many_gemms_mixed_widths_and_layouts(n, rows, x3):
    _run(_spec(n, n), rows, x3, seed=n)
