"""The constants helper of the boundary tests (kconst.py) finds every kernel constant the GPU tests name,
so a renamed constant fails here, on a CPU, instead of breaking the GPU run."""
import glob
import os
import re

from kconst import K, kernel_constants

TESTS = os.path.dirname(os.path.abspath(__file__))


def test_every_constant_the_gpu_tests_use_is_found():
    used = set()
    for path in glob.glob(os.path.join(TESTS, "test_gpu_*.py")):
        with open(path) as f:
            used |= set(re.findall(r"\bK\.(k\w+)", f.read()))
    assert used, "no GPU test names a kernel constant"
    missing = sorted(used - set(vars(K)))
    assert not missing, f"not found in kernels.cuh: {missing}"


def test_values_are_parsed_exactly(tmp_path):
    p = tmp_path / "k.cuh"
    p.write_text("constexpr uint32_t kA = 32;  // comment\n  constexpr uint32_t kB = 0xFFFFFFFFu;\n"
                 "constexpr uint8_t kC = 1;\nconstexpr uint32_t kD = 4096; \n")
    assert kernel_constants(str(p)) == {"kA": 32, "kB": 0xFFFFFFFF, "kD": 4096}
    assert K.kFatMin > 0 and K.kChunkBytes % 16 == 0 and K.kCmMaxBytes % K.kUnit == 0
