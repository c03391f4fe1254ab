"""The kernel contracts of tests/kernel_contract_cases.py on the GPU: every check with the CUDA kernels at the full case
set, the same check with the CPU emulation on identical inputs held against the kernel's result under the same
tolerance class (the emulation the CPU schedule tests trust matches the kernel), and run-to-run bit-exactness of the
kernels DESIGN.md §4 documents as free of floating-point atomics."""
import pytest
import torch

import kernel_contract_cases as KC
from multimodal_b200 import ops

pytestmark = pytest.mark.gpu

_ALL = [(op, c) for op, cases in KC.CASES.items() for c in cases]
_IDS = [f"{op}[{KC.case_id(c)}]" for op, c in _ALL]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("op,case", _ALL, ids=_IDS)
def test_kernel_meets_float64_contract_and_matches_emulation(dev, op, case):
    got = KC.CHECKS[op](ops, dev, case)
    torch.cuda.synchronize()
    emu = KC.CHECKS[op](KC.emulation(), "cpu", case)
    assert got.keys() == emu.keys()
    for name in got:
        slack = 0.0
        if name == "gsum":   # sums the stored g_bf16, whose elements may differ by one bf16 ulp between the two
            slack = (got["g_bf16"].got.double() - emu["g_bf16"].got.double()).abs().sum(0)
        KC.compare_recs(f"{op}.{name} kernel vs emulation", got[name], emu[name], slack)


_DET = [(op, c) for op, c in _ALL if op in KC.DETERMINISTIC]


@pytest.mark.parametrize("op,case", _DET, ids=[f"{op}[{KC.case_id(c)}]" for op, c in _DET])
def test_atomic_free_kernels_are_bit_exact_run_to_run(dev, op, case):
    a = KC.CHECKS[op](ops, dev, case)
    b = KC.CHECKS[op](ops, dev, case)
    for name in a:
        KC.assert_exact(f"{op}.{name} second run", b[name].got, a[name].got)

