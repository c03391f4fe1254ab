"""The kernel contracts of tests/kernel_contract_cases.py on the GPU: every check with the CUDA kernels at the full case
set, the same check with the CPU emulation on identical inputs held against the kernel's result under the same
tolerance class (the emulation the CPU schedule tests trust matches the kernel), run-to-run bit-exactness of the
kernels DESIGN.md §4 documents as free of floating-point atomics, and bit-identity of the two GEMM kernel variants."""
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
        slack, where = 0.0, None
        if name == "gsum":   # sums the stored g_bf16, whose elements may differ by one bf16 ulp between the two
            slack = (got["g_bf16"].got.double() - emu["g_bf16"].got.double()).abs().sum(0)
        if op == "gemm" and name == "colsum":   # sums the stored D0, likewise
            slack = (got["D0"].got.double() - emu["D0"].got.double()).abs().sum(0)
        if op == "gemm" and name == "D1":       # act of each one's own D0: compared where the two D0 agree
            where = KC._bits(got["D0"].got) == KC._bits(emu["D0"].got)
        KC.compare_recs(f"{op}.{name} kernel vs emulation", got[name], emu[name], slack, where)


_DET = [(op, c) for op, c in _ALL if op in KC.DETERMINISTIC]


@pytest.mark.parametrize("op,case", _DET, ids=[f"{op}[{KC.case_id(c)}]" for op, c in _DET])
def test_atomic_free_kernels_are_bit_exact_run_to_run(dev, op, case):
    a = KC.CHECKS[op](ops, dev, case)
    b = KC.CHECKS[op](ops, dev, case)
    for name in a:
        KC.assert_exact(f"{op}.{name} second run", b[name].got, a[name].got)


def _one_per_shape(op):
    seen = {}
    for c in KC.CASES[op]:
        base = {k: v for k, v in c.items() if k != "gemm_mode"}
        seen.setdefault(KC.case_id(base), base)
    return [(op, c) for c in seen.values()]


_FAMILY = [oc for op in KC.GEMM_FAMILY for oc in _one_per_shape(op)]


@pytest.mark.parametrize("op,case", _FAMILY, ids=[f"{op}[{KC.case_id(c)}]" for op, c in _FAMILY])
def test_gemm_variants_are_bit_identical(dev, op, case):
    """One CTA per 128 x 256 tile and 2-CTA clusters run the same wgmma sequence over the same k-blocks for every
    128-row block; only the tile origin and the B multicast differ, so every output is bit for bit the same."""
    a = KC.CHECKS[op](ops, dev, dict(case, gemm_mode=0))
    b = KC.CHECKS[op](ops, dev, dict(case, gemm_mode=1))
    assert a.keys() == b.keys()
    for name in a:
        KC.assert_exact(f"{op}.{name} cluster vs 1-CTA", b[name].got, a[name].got)
