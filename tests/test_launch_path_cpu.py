"""Every kernel launch goes through stb::launch (common.cuh, misc.cu).

The helper owns the launch policy: programmatic dependent launch, clusters, priority, the per-device opt-in to more than
the default dynamic shared memory, the launch count and the error check.  A `<<<>>>` launch, a hand-built launch
configuration, a function attribute or an SM count read anywhere else would keep a second copy of that policy (a
process-wide opt-in that misses a second device, for one)."""
import os

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stable-ts_b200", "csrc")
HOME = {"common.cuh", "misc.cu"}
FORBIDDEN = ["<<<", "cudaLaunchKernelEx", "cudaFuncSetAttribute", "cudaDevAttrMultiProcessorCount"]


def test_no_launch_policy_outside_the_helper():
    found = []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith(".cu") or name in HOME:
            continue
        with open(os.path.join(CSRC, name)) as f:
            text = f.read()
        found += [f"{name}: {tok}" for tok in FORBIDDEN if tok in text]
    assert not found, f"launch through stb::launch instead: {found}"
