"""CPU checks of the pair fusion rule (tc_pair_fuses, ovc_tcpack.h) through the kernel harness: which ResBlock conv
pairs the library runs as one kernel, and the ring of the C = 128 pair kernel."""
import importlib.util
import os

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def kc():
    spec = importlib.util.spec_from_file_location("kc_pair", os.path.join(HERE, "kernelcheck", "kc_pair.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.PairHarness()


def test_pair_fuses_generator_pairs(kc):
    """Every ResBlock pair of the C = 128 / 64 / 32 stages (k 3 / 7 / 11, dilation 1 / 3 / 5) is fused; the resident
    pairs tc_pair_fits accepts stay fused."""
    for C in (32, 64, 128):
        for K in (3, 7, 11):
            for D in (1, 3, 5):
                assert kc.pair_fuses(C, K, D), (C, K, D)
    for C, K in ((32, 3), (64, 3), (32, 5)):
        for D in (1, 3, 5):
            assert kc.pair_fits(C, K, D) and kc.pair_fuses(C, K, D), (C, K, D)


def test_pair_fuses_refusals(kc):
    assert not kc.pair_fuses(256, 3, 1)              # two column tiles: conv 2 would need a 256-wide operand
    assert not kc.pair_fuses(96, 3, 1)               # TN 32 with 3 column tiles
    assert not kc.pair_fuses(128, 3, 1, D2=3)        # conv 2 has dilation 1
    assert not kc.pair_fuses(128, 7, 1, K2=3)        # the same k
    assert not kc.pair_fuses(128, 3, 1, C2=64)
    assert not kc.pair_fuses(64, 3, 1, N1=128)
    assert not kc.pair_fuses(128, 13, 5)             # conv-1 halo 30 > 25
    assert kc.pair_fuses(32, 19, 1)                  # conv-2 halo 9: 128 + 18 rows = the on-chip operand
    assert not kc.pair_fuses(32, 21, 1)              # halo 10 does not fit


def test_pair_ring_slots(kc):
    # TN 128 pair: 1024 + 2 x 24 832 (A buffers) + 74 752 (conv-2 operand) + 12 x 8192 = 223 744 B <= 232 448
    assert kc.ring_slots(128, True) == 12
    assert 1024 + 2 * 24832 + 2 * (128 // 8) * 146 * 16 + kc.ring_slots(128, True) * 2 * 2 * 128 * 16 <= 232448
