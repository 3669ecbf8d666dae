"""CPU checks of the two-CTA-per-SM conv-pair configs (tc_pair_occ, ovc_tcpack.h) through the kernel harness: which
pairs run two CTAs per SM, that those configs fit half an SM's shared memory, that they keep every pair resident that
is resident at one CTA per SM, and that the two-CTA kernels compile without spills."""
import importlib.util
import os
import re

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SMEM_OCC2 = (233472 - 2 * 1024) // 2   # 228 KB per SM, less 1 KB reserved per CTA, halved


@pytest.fixture(scope="module")
def kc():
    spec = importlib.util.spec_from_file_location("kc_pair_occ", os.path.join(HERE, "kernelcheck", "kc_pair_occ.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.PairOccHarness()


def test_pair_occ_generator_table(kc):
    """The measured table: C = 32 k 3 / 7 and C = 64 k 7 / 11 run two CTAs per SM, the rest one."""
    want = {(32, 3): (2, 2), (32, 7): (2, 1), (32, 11): (1, 2), (64, 3): (1, 2), (64, 7): (2, 1), (64, 11): (2, 1),
            (128, 3): (1, 2), (128, 7): (1, 2), (128, 11): (1, 2)}
    for (C, K), (occ, nabuf) in want.items():
        for D in (1, 3, 5):
            cfg = kc.pair_occ(C, K, D)
            assert (cfg["occ"], cfg["nabuf"]) == (occ, nabuf), (C, K, D, cfg)


@pytest.mark.parametrize("C", [32, 64, 128])
def test_pair_occ_budget_and_residency(kc, C):
    """Every fused pair: a two-CTA config fits SMEM_OCC2 and its ring holds every slot of a pair it marks resident;
    a pair resident at one CTA per SM stays resident."""
    for K in range(3, 20, 2):
        for D in (1, 3, 5):
            if not kc.pair_fuses(C, K, D):
                continue
            cfg = kc.pair_occ(C, K, D)
            n_w = 2 * (C // 16) * K
            slot = 2 * 2 * C * 16
            a2 = 2 * (C // 8) * 146 * 16
            assert cfg["smem"] == 1024 + cfg["nabuf"] * 24832 + a2 + cfg["ring"] * slot, (C, K, D, cfg)
            assert cfg["resident"] == (n_w <= cfg["ring"]), (C, K, D, cfg)
            if cfg["occ"] == 2:
                assert cfg["smem"] <= SMEM_OCC2, (C, K, D, cfg)
                assert C in (32, 64), (C, K, D, cfg)
            if n_w <= kc.ring_slots(C, True):
                assert cfg["resident"], (C, K, D, cfg)


def test_pair_occ2_kernels_no_spills():
    """ptxas report of the library build: the two-CTA pair kernels use at most 80 registers (384 threads x 2 CTAs)
    and spill nothing."""
    log = os.path.join(ROOT, "openvoice_b200", "csrc", "build", "ovc_lib.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log: build the library with `make -C openvoice_b200/csrc`")
    text = open(log).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(_ZN3ovc13tcconv_kernelILi(\d+)ELb1ELi2ELi(\d)E\w*)' for 'sm_90a'\n"
                         r"(?:ptxas info[^\n]*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill "
                         r"loads\nptxas info\s*: Used (\d+) registers", text):
        C, nabuf, stack, st, ld, regs = (int(g) for g in m.groups()[1:])
        found[(C, nabuf)] = (stack, st, ld, regs)
    assert set(found) == {(32, 2), (32, 1), (64, 1)}, found
    for key, (stack, st, ld, regs) in found.items():
        assert st == 0 and ld == 0 and regs <= 80, (key, found[key])
