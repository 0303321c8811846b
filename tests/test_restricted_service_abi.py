"""The restricted query service's C ABI refuses bad handles and arguments without a device, and its C++ mirror
(helix::RestrictedSearchService in host/vector_index.hpp) compiles against the header."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest

import helix_db_b200 as hx

ROOT = Path(__file__).resolve().parent.parent


def _cfg(k=10, **kw):
    c = hx._ServiceConfig()
    c.k = k
    for f, v in kw.items():
        setattr(c, f, v)
    return c


def test_null_index_handle_is_index_not_found():
    lib = hx.load_library()
    h = C.c_void_p()
    assert lib.hx_restricted_service_create(None, C.byref(_cfg()), 0, C.byref(h)) == hx.HX_ERR_INDEX_NOT_FOUND


def test_null_arguments_and_bad_config_are_invalid_parameter():
    lib = hx.load_library()
    # an index handle the checks below never dereference: they all fail before the device is touched
    fake = C.create_string_buffer(4096)
    ix = C.cast(fake, C.c_void_p)
    h = C.c_void_p()
    assert lib.hx_restricted_service_create(ix, None, 0, C.byref(h)) == hx.HX_ERR_INVALID_PARAMETER
    assert lib.hx_restricted_service_create(ix, C.byref(_cfg()), 0, None) == hx.HX_ERR_INVALID_PARAMETER
    for bad in (_cfg(k=0), _cfg(k=801), _cfg(ef=50), _cfg(ctas_per_sm=1), _cfg(cta_warps=4), _cfg(rows_in_flight=2),
                _cfg(visited_log2=12)):
        assert lib.hx_restricted_service_create(ix, C.byref(bad), 0, C.byref(h)) == hx.HX_ERR_INVALID_PARAMETER
    assert lib.hx_restricted_service_create(ix, C.byref(_cfg()), 999_999, C.byref(h)) == hx.HX_ERR_INVALID_PARAMETER
    q = (C.c_float * 4)()
    ids = (C.c_uint64 * 2)(1, 2)
    t = C.c_uint64()
    out_i = (C.c_uint64 * 10)()
    out_s = (C.c_float * 10)()
    cnt = C.c_uint32()
    assert lib.hx_service_submit_restricted(None, q, ids, 2, C.byref(t)) == hx.HX_ERR_INVALID_PARAMETER
    assert lib.hx_service_submit_restricted_set(None, q, None, C.byref(t)) == hx.HX_ERR_INVALID_PARAMETER
    assert lib.hx_service_search_restricted(None, q, ids, 2, out_i, out_s, C.byref(cnt)) == hx.HX_ERR_INVALID_PARAMETER
    assert lib.hx_service_search_restricted_set(None, q, None, out_i, out_s, C.byref(cnt)) == hx.HX_ERR_INVALID_PARAMETER


def test_cpp_restricted_service_mirror_compiles_against_the_header(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    src = tmp_path / "t.cpp"
    src.write_text('#include "%s"\n'
                   'int use(hx_index* ix, hx_candidates* set) {\n'
                   '  helix::RestrictedSearchService s(ix, 10, 2000000);\n'
                   '  std::vector<float> q(8, 1.0f);\n'
                   '  auto r = s.search(q, helix::RestrictedVectorCandidates::from_ids({3, 1, 2}));\n'
                   '  uint64_t t = s.submit(q.data(), set);\n'
                   '  uint64_t ids[10]; float sc[10]; uint32_t n = 0;\n'
                   '  return (int)r.size() + (s.poll(t, ids, sc, &n) ? 1 : 0);\n'
                   '}\nint main() { return 0; }\n' % (ROOT / "helix-db_b200" / "host" / "vector_index.hpp"))
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
