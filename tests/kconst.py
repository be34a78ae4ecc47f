"""The kernels' threshold constants, read from the `constexpr uint32_t kName = value;` lines of
push-cdn_b200/csrc/kernels.cuh, so that boundary tests place their cases around the values the kernels
were built with and follow any retuning.  Use as `K.kCmMaxBytes`; an unknown name raises."""
import os
import re
import types

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "push-cdn_b200", "csrc", "kernels.cuh")
_CONSTEXPR = re.compile(r"^\s*constexpr\s+uint32_t\s+(k\w+)\s*=\s*(0[xX][0-9A-Fa-f]+|\d+)[uU]?\s*;", re.M)


def kernel_constants(path: str = HEADER) -> dict:
    with open(path) as f:
        return {name: int(v, 0) for name, v in _CONSTEXPR.findall(f.read())}


K = types.SimpleNamespace(**kernel_constants())
