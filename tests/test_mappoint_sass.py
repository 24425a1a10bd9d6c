"""The map-point kernels in geom.cu: present in the disassembly, and the add kernel's explicit FFMAs are exactly the sixteen
A-row FMAs of the one triangulate it inlines (every other FFMA / DFMA of geom.cu is audited by tests/test_geom_sass.py)."""
import re

from tests.test_geom_sass import SRC, fma_sites  # noqa: F401  (fma_sites is the module-scoped disassembly fixture)


def _named(sites, name):
    return [s for s in sites if re.search(rf"{len(name)}{name}E", s[0])]


def test_map_point_kernels_are_present(fma_sites):  # noqa: F811
    # the add and erase kernels carry the rounded division sequences, so both show up among the FMA sites
    for name in ("k_mp_add", "k_mp_erase"):
        assert _named(fma_sites, name), name


def test_add_kernel_fmas_are_the_sixteen_a_row_fmas(fma_sites):  # noqa: F811
    src = open(SRC).read().splitlines()
    fma_lines = {i + 1 for i, t in enumerate(src) if "__fmaf_rn" in t}
    add = _named(fma_sites, "k_mp_add")
    assert sum(1 for _, in_sub, op, line in add if not in_sub and op == "FFMA" and line in fma_lines) == 16
    for name in ("k_mp_erase", "k_mp_update_measure", "k_mp_check"):
        assert not any(line in fma_lines for _, _, _, line in _named(fma_sites, name)), name
