"""What the fp64 kernel sweeps (test_gemm_plans_gpu.py, test_norm_sweep_gpu.py, test_attention_sweep_gpu.py) share:
recording the ops calls of a workload, the fp16 spacing, the failure tally of one sweep title and the branch-coverage
check. Each sweep keeps its own signatures, operands, references, bounds and dispatch mirror."""
import time

import pytest
import torch

import helpers  # noqa: F401  (puts the repository on sys.path)
from sdb200 import ops

NAN = float("nan")
GUARD = 16         # NaN elements before and after every output


def ulp16(x):
    """Spacing of fp16 numbers at |x| (subnormal spacing below 2^-14)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def eoff(t):
    """Element offset of t's data from the nearest 16-byte boundary."""
    return (t.data_ptr() % 16) // t.element_size()


def signature(p):
    """A problem dict as a hashable tuple: two calls are one problem when their dicts are equal."""
    return tuple(sorted(p.items()))


def record(workload, dev, sigs):
    """Runs workload(dev) once under no_grad with the autotuner off and each ops function named in sigs wrapped.
    sigs[name] turns the arguments of one call into a problem dict. Returns (number of calls, the distinct problems of
    all wrapped functions together in first-call order): the sweeps seed each problem's operands by its index."""
    calls, seen, problems = 0, set(), []

    def wrap(name, fn):
        def rec(*a, **kw):
            nonlocal calls
            p = sigs[name](*a, **kw)
            calls += 1
            key = signature(p)
            if key not in seen:
                seen.add(key)
                problems.append(p)
            return fn(*a, **kw)
        return rec

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "AUTOTUNE", False)
        mp.setattr(ops, "TUNED", {})
        for name in sigs:
            mp.setattr(ops, name, wrap(name, getattr(ops, name)))
        with torch.no_grad():
            workload(dev)
        torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return calls, problems


class Tally:
    """Failure rows, launch count and wall time of one sweep title (a workload or a synthetic group)."""

    def __init__(self, title, columns="problem, check, value"):
        self.title, self.columns, self.failures, self.launches, self.t0 = title, columns, [], 0, time.time()

    def finish(self, n_problems, summary):
        """Prints the title's counts, time and `summary` (the sweep's calibration), then fails with the table."""
        torch.cuda.synchronize()
        print(f"\n{self.title}: {n_problems} problems, {self.launches} launches, {time.time() - self.t0:.1f} s; {summary}")
        if self.failures:
            rows = "\n".join(" | ".join(map(str, f)) for f in self.failures[:200])
            pytest.fail(f"{self.title}: {len(self.failures)} failing ({self.columns}):\n{rows}")


def check_coverage(cover, required, kernel):
    """Every class in `required` was launched by the sweeps of this session (skips when none of them ran)."""
    if not cover:
        pytest.skip(f"the {kernel} sweeps did not run in this session")
    print("\ncoverage: " + ", ".join(f"{k} {cover[k]}" for k in sorted(cover)))
    assert required <= set(cover), sorted(required - set(cover))
