"""The C-ABI library loads on a CPU-only box and exports every entry point include/igmc_b200.h declares
(no compute calls: those need a GPU)."""
import ctypes
import os
import re

from igmc_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "igmc_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\bint\s+(igmc_[a-z_0-9]+)\s*\(", src)))


def test_header_symbols_are_exported_and_bound():
    names = declared_symbols()
    assert len(names) >= 10
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), "missing export %s" % n
    # the ctypes binding covers exactly the declared surface
    assert sorted(_lib.EXPORTS) == names


def test_build_info_and_plans():
    lib = _lib.load()
    assert lib.igmc_build_info() == 90
    from igmc_b200.models import IGMC
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)
    c = ctypes.byref(m._cmodel)
    for n_cap, cl in ((202, 1), (202, 2), (202, 3), (202, 4), (402, 2), (402, 0), (202, 0)):
        f, b = lib.igmc_model_plan(c, n_cap, cl, 0), lib.igmc_model_plan(c, n_cap, cl, 1)
        assert 0 < f <= 227 * 1024 and 0 < b <= 227 * 1024, (n_cap, cl, f, b)
    assert lib.igmc_model_plan(c, 5000, 1, 0) < 0          # does not fit: refused, never silently clipped
    assert lib.igmc_model_plan(c, 202, 5, 0) < 0           # unsupported cluster size
    # the list image of a plan: shape only (no device memory touched)
    img = _lib.Stage()
    assert lib.igmc_stage_plan(c, 202, 2, 1, ctypes.byref(img)) == 0
    assert img.cluster == 2 and img.chunk % 16 == 0 and img.lcap % 4 == 0 and img.tab_ints % 4 == 0
    assert lib.igmc_raw_grad_count(c) == 800 + 3 * 6176    # per layer (R+1)*inp*32 + 32 floats
    m30 = IGMC(4, latent_dim=[32] * 4, num_relations=30, num_bases=4, regression=True)
    assert lib.igmc_model_plan(ctypes.byref(m30._cmodel), 100, 2, 0) < 0   # relation-space plan needs R <= 12
    assert lib.igmc_model_plan(ctypes.byref(m30._cmodel), 100, 0, 0) > 0   # generic plan takes it


def test_reduce_update_grid_blocks():
    """the grid of the fused reduce -> all-reduce -> Adam kernel, one block per layer input row plus the readout
    parameters, for in0 = 4 (R and NB do not enter), without a device.  Two blocks per SM hold 264 on a 132-SM H100:
    from 5 layers on the engine takes the separate kernels"""
    from igmc_b200.models import IGMC
    want = {1: 38, 2: 102, 3: 166, 4: 230, 5: 294, 6: 358, 7: 422, 8: 486}
    lib = _lib.load()
    for L, blocks in want.items():
        for R, NB in ((5, 4), (12, 2)):
            m = IGMC(4, latent_dim=[32] * L, num_relations=R, num_bases=NB, regression=True)
            got = ctypes.c_int(-1)
            assert lib.igmc_reduce_update_grid(ctypes.byref(m._cmodel), ctypes.byref(got), None) == 0
            assert got.value == blocks, (L, R, NB, got.value)


def test_struct_sizes_match_header_layout():
    # pointer-sized fields and 4-byte ints exactly as declared (guards against a silent ABI drift)
    P = ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.CSR) == 5 * P + 8
    assert ctypes.sizeof(_lib.Pairs) == 5 * P
    assert ctypes.sizeof(_lib.ExtractWS) == 9 * P
    assert ctypes.sizeof(_lib.Adj) == 7 * P + 8
    assert ctypes.sizeof(_lib.Model) == 4 * (4 + 4 * 8 + 4 + 2 + 1 + 1 + 1)
    assert ctypes.sizeof(_lib.Stage) == 3 * P + 16
    assert ctypes.sizeof(_lib.SortPool) == 4 * 19
    assert ctypes.sizeof(_lib.SortPoolSaved) == 10 * P
