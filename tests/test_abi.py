"""CPU tests of the boundary: the C-ABI library builds, loads, exports every symbol the header declares,
and refuses to compute without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    import vectordb_b200
    if not os.path.exists(vectordb_b200.library_path()):
        from vectordb_b200.lib import build_library
        build_library()
    return vectordb_b200.load_library()


def test_header_symbols_exported():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    declared = sorted(set(re.findall(r"EPS_API[^;(]*?\b(eps_[a-z_0-9]+)\s*\(", hdr)))
    assert len(declared) >= 19
    for name in declared:
        assert hasattr(L, name), "symbol %s declared in include/epsilla_b200.h but not exported" % name
    from vectordb_b200.lib import EXPORTS
    assert sorted(EXPORTS) == declared


def test_struct_layouts_match_header():
    from vectordb_b200.lib import BuildParams, FilterNode, StatsStruct
    assert C.sizeof(FilterNode) == 64
    assert C.sizeof(StatsStruct) == 72
    assert C.sizeof(BuildParams) == 48


def test_no_cpu_fallback_without_gpu():
    import vectordb_b200
    L = _lib()
    if L.eps_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(vectordb_b200.EpsError) as e:
        vectordb_b200.Index("l2", 8, host_vectors=np.zeros((4, 8), np.float32))
    assert e.value.code == 50001  # EPS_ERR_NO_DEVICE
    from vectordb_b200.index import pair_distances
    with pytest.raises(vectordb_b200.EpsError):
        pair_distances("l2", np.zeros((1, 4), np.float32), np.zeros((1, 4), np.float32))
    import ctypes as C
    h = C.c_void_p()
    assert L.eps_index_create_view(None, C.byref(h)) != 0 and not h.value  # argument check before any device work


def test_product_does_not_import_oracle():
    """The product package must never import, link or execute anything under oracle/ (tier rule 3)."""
    pkg = os.path.join(ROOT, "vectordb_b200")
    bad = re.compile(r"(from\s+oracle|import\s+oracle|oracle/|oracle\.oracle|libepsilla_port|libepsilla_ref|oracle_port)")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")) or f == "Makefile":
                src = open(os.path.join(dp, f), errors="replace").read()
                m = bad.search(src)
                assert m is None, "%s references the oracle: %r" % (f, m.group(0))


def test_header_is_plain_c(tmp_path):
    """The boundary is a C ABI: the header must compile as strict C99 (no C++ / torch types) and link against the
    library by symbol name."""
    import subprocess
    src = tmp_path / "abi.c"
    src.write_text(
        '#include "epsilla_b200.h"\n'
        "#include <stddef.h>\n"
        "int main(void) {\n"
        "  eps_filter_node n; eps_stats s; eps_build_params b; eps_index* ix = NULL;\n"
        "  (void)n; (void)s; (void)b;\n"
        "  if (sizeof(eps_filter_node) != 64 || sizeof(eps_stats) != 72) return 2;\n"
        "  /* no device in this container: creation must fail loudly, never fall back */\n"
        "  return eps_index_create(&ix, EPS_METRIC_L2, 8, NULL, 0, 0) == EPS_OK && eps_device_count() == 0 ? 3 : 0;\n"
        "}\n")
    exe = tmp_path / "abi"
    lib_dir = os.path.join(ROOT, "vectordb_b200")
    _lib()
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           str(src), "-o", str(exe), "-L", lib_dir, "-lepsilla_b200", "-Wl,-rpath," + lib_dir])
    assert subprocess.call([str(exe)]) == 0


def test_dropin_library_binds_reference_symbols_to_the_gpu_path():
    """oracle/_ref/dropin/libepsilla_ref_b200.so = the reference's own objects with three symbols replaced: each must be
    defined exactly once (strong), and the library must import the C ABI from libepsilla_b200.so (no CPU body left)."""
    import subprocess
    so = os.path.join(ROOT, "oracle", "_ref", "dropin", "libepsilla_ref_b200.so")
    if not os.path.exists(so):
        pytest.skip("drop-in not built (needs a reference checkout at build time)")
    dyn = subprocess.check_output(["nm", "-D", "-C", so], text=True)
    for sym in ("VecSearchExecutor::Search(", "VecSearchExecutor::VecSearchExecutor(long, long,",
                "ANNGraphSegment::BuildFromVectorTable("):
        strong = {l.split()[0] for l in dyn.splitlines() if sym in l and " T " in l}
        weak = [l for l in dyn.splitlines() if sym in l and " W " in l]
        assert len(strong) == 1 and not weak, (sym, strong, weak)
    for imp in ("eps_search_batch", "eps_index_build", "eps_index_get_graph", "eps_index_set_graph", "eps_index_sync_rows"):
        assert any(l.strip().startswith("U " + imp) for l in dyn.splitlines()), imp
    needed = subprocess.check_output(["readelf", "-d", so], text=True)
    assert "libepsilla_b200.so" in needed
