"""The C-ABI library loads without a GPU and exports every symbol include/helix_b200.h declares."""
import ctypes
import re
from pathlib import Path

import pytest

import helix_db_b200 as hx

ROOT = Path(__file__).resolve().parent.parent


def declared_symbols():
    text = (ROOT / "include" / "helix_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(hx_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_list_agree():
    assert declared_symbols() == sorted(hx.ABI_SYMBOLS)


def test_library_exports_every_declared_symbol():
    lib = hx.load_library()
    for name in declared_symbols():
        assert hasattr(lib, name), f"libhelix_b200.so does not export {name}"
    assert b"sm_90a" in lib.hx_version()


def test_no_torch_or_oracle_in_the_product_library():
    # the boundary is plain C: no torch types, and the oracle is never linked into the product
    import subprocess
    out = subprocess.run(["ldd", str(hx.LIB_PATH)], capture_output=True, text=True).stdout
    assert "torch" not in out and "hx_oracle" not in out
    syms = subprocess.run(["nm", "-D", "--defined-only", str(hx.LIB_PATH)], capture_output=True, text=True).stdout
    assert "hxo_" not in syms


def test_product_sources_never_reference_the_oracle():
    for p in (ROOT / "helix-db_b200").rglob("*"):
        if p.suffix in {".cu", ".cuh", ".hpp", ".h", ".py", ".sh"}:
            t = p.read_text()
            assert "hx_oracle" not in t and "import hxo" not in t and "from oracle" not in t, p


def test_pure_entry_points_work_without_a_device():
    lib = hx.load_library()
    assert hx.restricted_plan(256, 128) == "Exact"          # restricted.rs:40-42,433-440
    assert hx.restricted_plan(257, 128) == "FilteredGraph"
    assert hx.restricted_plan(256, 4096) == "Exact"
    assert hx.restricted_plan(256, 4097) == "FilteredGraph"
    assert lib.hx_search(None, None, 0, None, None, None, None, None) == hx.HX_ERR_INDEX_NOT_FOUND


def test_product_path_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(hx.HelixDbError) as e:
        hx.VectorIndex(hx.Metric.Euclidean, hx.VectorIndexConfig("t", "embedding", 8))
    assert e.value.code == hx.HX_ERR_CUDA and "no CPU fallback" in str(e.value)


def test_policy_defaults_and_order_code_without_a_device():
    import ctypes as C
    lib = hx.load_library()
    p = hx._PolicyParams()
    lib.hx_policy_params_default(C.byref(p))                 # SearchParams::new (mod.rs:482-500)
    assert (p.bypass_min_frontier, p.bypass_window_expansions, p.read_budget_multiplier) == (24, 4, 3)
    assert abs(p.bypass_min_filter_rate - 0.12) < 1e-7 and p.sampling_ratio_override < 0 and p.failure_prob_override < 0
    assert lib.hx_order_code_from_simhash_bits(0) == 0       # simhash.rs:313-330
    assert lib.hx_order_code_from_simhash_bits(2**64 - 1) == 2**64 - 1
    for shift, bit in ((63, 63), (47, 62), (31, 61), (15, 60)):
        assert lib.hx_order_code_from_simhash_bits(1 << shift) == 1 << bit
    sp = hx.SearchParams.new(10)
    assert sp.requires_query_simhash() and sp._c().pre_sampling_ratio < 0          # Option::None travels as a negative
    assert not hx.SearchParams.strict(10).requires_query_simhash()
    t = hx.SearchParams.throughput_profile_floor_92(10)
    assert t.ef() == 48 and abs(t._c().pre_sampling_ratio - 0.20) < 1e-7


def test_cpp_host_mirror_compiles_against_the_header(tmp_path):
    # helix-db_b200/host/vector_index.hpp is the C++ host side a non-Python caller links: it must follow the C ABI header
    import shutil
    import subprocess
    if shutil.which("g++") is None:
        import pytest
        pytest.skip("g++ not available")
    src = tmp_path / "t.cpp"
    src.write_text('#include "%s"\nint main() { helix::SearchParams p(10); p.with_simhash_failure_prob(0.2f)'
                   '.with_simhash_bypass_tuning(24, 4, 0.12f, 3); return p.raw().k == 10 && !helix::SearchParams::strict(3)'
                   '.requires_query_simhash() ? 0 : 1; }\n' % (ROOT / "helix-db_b200" / "host" / "vector_index.hpp"))
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_cpp_host_mirror_links_and_runs(tmp_path):
    """The C++ host mirror is not only parsed: tests/cpp/host_mirror_selftest.cpp is linked against libhelix_b200.so and
    executed.  Without a GPU its device-free half runs (SearchParams / candidate-set contracts of the reference, the pure
    ABI entry points) and the constructor must refuse with "no CPU fallback"; tests/test_gpu_parity.py runs the same
    binary on the device."""
    import shutil
    import torch
    from hx_testutil import build_and_run_cpp_selftest
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    rc, out = build_and_run_cpp_selftest(tmp_path)
    assert rc == 0, out
    if not torch.cuda.is_available():
        assert "device-free checks passed" in out, out


def test_index_config_is_validated_before_the_device_is_touched():
    """Connections / Layer0Connections / ConstructionBeamWidth (parameters.rs:25-100, config/indexes.rs:411-466): m is
    non-zero and both m0 and ef_construction must cover it -> InvalidVectorConfig, with or without a GPU."""
    def make(**kw):
        cfg = hx.VectorIndexConfig("t", "embedding", kw.pop("dimension", 8))
        cfg.m, cfg.m0, cfg.ef_construction = kw.get("m", 16), kw.get("m0", 32), kw.get("efc", 200)
        return hx.VectorIndex(hx.Metric.Cosine, cfg)
    for bad in (dict(m=0), dict(m=16, m0=15), dict(m=16, efc=15), dict(dimension=0), dict(m=64)):   # m=64 > default m0=32
        with pytest.raises(hx.HelixDbError) as e:
            make(**bad)
        assert e.value.variant == "InvalidVectorConfig", bad


def test_product_plan_and_budget_functions_match_the_reference_literals():
    """The PRODUCT's device-free planning entry points (not the oracle's): hx_restricted_plan and hx_filtered_budgets against
    the literals of the reference's admission test (tests/production_support/vector/restricted.rs:459-530)."""
    import ctypes as C
    lib = hx.load_library()
    assert hx.restricted_plan(256, 1536) == "Exact" and hx.restricted_plan(256, 5000) == "FilteredGraph"
    assert hx.restricted_plan(257, 2) == "FilteredGraph" and hx.restricted_plan(1000, 1536) == "FilteredGraph"
    for percent, want in ((100, 100), (150, 150), (200, 200), (400, 400), (0, 150)):   # 0 = FILTERED_BEAM_PERCENT
        b = hx.FilteredBudgets()
        lib.hx_filtered_budgets(10, 100, percent, 1000, C.byref(b))
        assert b.ef_filtered == want and (b.sampled_seeds, b.vector_payloads) == (64, 800)
        assert (b.routing_rows, b.bridge_rows) == (want * 16, want * 8)
    b = hx.FilteredBudgets()
    lib.hx_filtered_budgets(800, 800, 150, 1000, C.byref(b))
    assert b.vector_payloads == 800                             # MAX_RESTRICTED_RESULT_COUNT == the payload budget
    lib.hx_filtered_budgets(10, 100, 150, 40, C.byref(b))
    assert (b.ef_filtered, b.sampled_seeds, b.vector_payloads) == (40, 40, 40)   # everything clamps to |C|
