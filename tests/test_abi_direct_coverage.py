"""CPU: every entry point include/mmx.h declares is called directly by some GPU test (tests/test_*_gpu.py), or is listed
below with the test that exercises it another way.  A new entry point without a test fails here."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# entry points reached through a Python wrapper or an engine object, or plain library state: where they are tested
INDIRECT = {
    "mmx_version": "test_capi.py (CPU) and build()",
    "mmx_last_error": "library state: its text is the message of every MmxError the GPU tests raise",
    "mmx_profile_gemm": "bench.py's GEMM roofline line: timing only, no result to compare",
    "mmx_profile_gemm_report": "bench.py's GEMM roofline line: timing only, no result to compare",
    "mmx_gemm_trace": "profiling aid (profiles/attn_trace.py); it only sets a pointer",
    "mmx_memcpy_d2d": "through ClipEngine.tap, test_clip_gpu.py",
    "mmx_linear": "mmx_linear_packed with packed = NULL, test_primitives_gpu.py",
    "mmx_linear_dgrad": "mmx_linear_dgrad_packed with packed = NULL, test_primitives_gpu.py",
    "mmx_clip_create": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_destroy": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_load_tensor": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_finalize": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_interpret_device": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_interpret_host": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_set_serial": "ClipEngine object, test_clip_gpu.py",
    "mmx_clip_tap": "ClipEngine object, test_clip_gpu.py",
}


def _declared():
    text = open(os.path.join(ROOT, "include", "mmx.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mmx_[a-z0-9_]+)\s*\(", text)))


def _called_in_gpu_tests():
    called = set()
    for path in glob.glob(os.path.join(ROOT, "tests", "test_*_gpu.py")):
        called |= set(re.findall(r"\.(mmx_[a-z0-9_]+)\s*\(", open(path).read()))
    return called


def test_every_entry_point_has_a_test():
    declared, called = _declared(), _called_in_gpu_tests()
    assert len(declared) >= 60
    missing = [s for s in declared if s not in called and s not in INDIRECT]
    assert not missing, f"entry points with no direct call in tests/test_*_gpu.py and no INDIRECT entry: {missing}"


def test_allowlist_is_current():
    """An INDIRECT entry names a declared symbol that no GPU test calls directly (otherwise it is stale)."""
    declared, called = set(_declared()), _called_in_gpu_tests()
    assert not set(INDIRECT) - declared, sorted(set(INDIRECT) - declared)
    assert not set(INDIRECT) & called, sorted(set(INDIRECT) & called)
    assert all(reason.strip() for reason in INDIRECT.values())
