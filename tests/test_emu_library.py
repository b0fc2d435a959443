"""The whole C-ABI library on the CPU: `tests/emu/build_emu_lib.py` compiles the PRODUCT sources
(distributed_faiss_b200/csrc/*.cu, host drivers included) with g++ on top of the fiber SIMT
runtime, and a subset of the `gpu` parity tests is run against that build in a subprocess
(DFX_EMU_LIB, see tests/conftest.py).  This is how host-side changes and the experimental kernel
kernels are checked in a container without a GPU: same
sources, same tests, same oracle; only the PTX primitives (dfx_ptx.cuh) and the wgmma screening
kernel (its result is restated in C++; everything around it is the product code) are not what runs
on hardware.

The full `-m gpu` suite also passes this way but takes tens of minutes; the subset below is sized
for the regular CPU run.  Run everything with:
    DFX_EMU_LIB=$(python tests/emu/build_emu_lib.py) DFX_EXPERIMENTAL=1 python -m pytest tests -m gpu
"""
import os
import platform
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SUBSET = [
    "tests/test_gpu_parity.py::test_flat_matches_oracle[7-1]",
    "tests/test_gpu_parity.py::test_flat_edge_cases",
    "tests/test_gpu_parity.py::test_ivf_matches_oracle[oracle-ivf_flat-0-64-16-0]",
    "tests/test_gpu_parity.py::test_ivf_matches_oracle[oracle-ivf_pq-1-128-32-32]",
    "tests/test_gpu_parity.py::test_ivf_matches_oracle[oracle-ivf_pq-1-96-16-24]",
    "tests/test_gpu_parity.py::test_ivf_matches_oracle[oracle-ivf_sq-1-64-16-0]",
    "tests/test_gpu_parity.py::test_ivf_edge_cases",
    "tests/test_gpu_parity.py::test_merge_reference_golden",
    "tests/test_gpu_parity.py::test_merge_matches_oracle[8-64-10]",
    "tests/test_gpu_parity.py::test_exchange_kernels_match_numpy",    # packed merge, encode, filter, owner decode
    "tests/test_gpu_parity.py::test_interleaved_and_row_major_pq_layouts_agree",
    "tests/test_gpu_parity.py::test_block_scan_matches_oracle",   # K3 + K4 fused block scan
    "tests/test_gpu_api.py::test_sharded_equals_unsharded_exactly",   # servers + client over the C-ABI
    "tests/test_gpu_api.py::test_result_aggregation_on_device",
    # coarse quantizer through the tensor-core path: screening restated in C++ (dfx_tc.cu, DFX_EMU),
    # group selection + exact re-rank + drivers are the product code
    "tests/test_gpu_parity.py::test_tensor_core_coarse_quantizer_matches_oracle[ivf_flat-1-64-0]",
    "tests/test_gpu_parity.py::test_flat_tensor_core_path_matches_oracle[0]",    # flat_tensor_cores=1
    "tests/test_gpu_parity.py::test_flat_tensor_core_path_matches_oracle[1]",
    # more near-ties than kept groups -> exact fallback; AUTO screening precision follows the data
    "tests/test_gpu_parity.py::test_tensor_core_near_tie_overflow_is_redone_exactly",
    "tests/test_gpu_parity.py::test_tensor_core_many_groups_select_from_all_candidates",   # rerank_kernel<0> + select
    "tests/test_gpu_parity.py::test_tensor_core_auto_precision_follows_the_data",
]


def test_gpu_parity_subset_on_the_emulated_library():
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    lib = build_emu_lib.build()
    env = dict(os.environ, DFX_EMU_LIB=lib, DFX_EXPERIMENTAL="1")
    run = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + SUBSET,
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (run.stdout + run.stderr)[-3000:]
    assert run.returncode == 0, tail
    assert f"{len(SUBSET)} passed" in run.stdout, tail


def test_fuzz_smoke_on_the_emulated_library():
    """a few seconds of tests/emu/fuzz_against_oracle.py (random shapes, kinds, chunked adds, kernel
    variants) -- the long runs are done by hand with the AddressSanitizer build"""
    if shutil.which("g++") is None or platform.machine() != "x86_64":
        pytest.skip("the emulator needs g++ on x86-64")
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        import build_emu_lib
    finally:
        sys.path.pop(0)
    env = dict(os.environ, DFX_EMU_LIB=build_emu_lib.build())
    run = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emu", "fuzz_against_oracle.py"), "1000", "12"],
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0 and "0 failures" in run.stdout, (run.stdout + run.stderr)[-3000:]
