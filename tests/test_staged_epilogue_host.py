"""CPU checks of the staged-epilogue kernels (tcconv_kernel<128, PAIR, 1, 2, true>, OVC_OPT_STAGED_EPI) through the kernel
harness: block size, shared-memory and register budget, where the staging tile lives, and that ptxas spills nothing."""
import ctypes as C
import importlib.util
import os
import re

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SMEM_MAX = 232448   # 227 KB of opt-in shared memory per CTA (sm_90)


@pytest.fixture(scope="module")
def kc():
    spec = importlib.util.spec_from_file_location("kc", os.path.join(HERE, "kernelcheck", "kc.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    h = m.Harness(os.path.join(HERE, "kernelcheck", "libovc_kc_staged.so"))
    h.lib.kc_staged_cfg.argtypes = [C.c_int, C.c_void_p]
    return h


def cfg(kc, pair):
    out = (C.c_longlong * 8)()
    kc.lib.kc_staged_cfg(int(pair), C.cast(out, C.c_void_p))
    return dict(zip(("threads", "smem", "stage", "sbuf", "a2", "prod", "mma", "store"), out))


@pytest.mark.parametrize("pair", [False, True])
def test_staged_budget(kc, pair):
    """512 threads; the staging tile holds a tile's 128 x 128 fp32 results; producers, MMA and store warpgroups use
    exactly the 64 K registers of an SM; the shared memory fits one CTA per SM."""
    c = cfg(kc, pair)
    assert c["threads"] == 512, c
    assert c["stage"] == 128 * 128 * 4, c
    assert 128 * c["prod"] + 256 * c["mma"] + 128 * c["store"] == 65536, c
    assert all(r % 8 == 0 and 24 <= r <= 256 for r in (c["prod"], c["mma"], c["store"])), c
    assert c["smem"] <= SMEM_MAX, c
    if pair:
        # the pair stages in its conv-2 operand: no extra shared memory
        assert c["sbuf"] == 0 and c["stage"] <= c["a2"] == 2 * 16 * 146 * 16, c
        assert c["smem"] == 1024 + 2 * 24832 + c["a2"] + 12 * 2 * 2 * 128 * 16, c
    else:
        assert c["sbuf"] == c["stage"], c
        assert c["smem"] == 1024 + 2 * 24832 + 12 * 2 * 2 * 128 * 16 + c["stage"], c


def test_stage_pays(kc):
    """The library stages split-precision convs and pairs of k >= 5 only (single pass and k = 1 / 3 measured slower)."""
    for K in (1, 3, 5, 7, 11):
        assert kc.lib.kc_stage_pays(K, 3) == (K >= 5), K
        assert kc.lib.kc_stage_pays(K, 1) == 0, K


def test_staged_kernels_no_spills():
    """ptxas report of the library build: both staged kernels spill nothing (one CTA of 512 threads per SM)."""
    log = os.path.join(ROOT, "openvoice_b200", "csrc", "build", "ovc_lib.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log: build the library with `make -C openvoice_b200/csrc`")
    text = open(log).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(_ZN3ovc13tcconv_kernelILi128ELb(\d)ELi1ELi2ELb1E\w*)' for 'sm_90a'\n"
                         r"(?:ptxas info[^\n]*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill "
                         r"loads\nptxas info\s*: Used (\d+) registers", text):
        pair, stack, st, ld, regs = (int(g) for g in m.groups()[1:])
        found[pair] = (stack, st, ld, regs)
    assert set(found) == {0, 1}, found
    for key, (stack, st, ld, regs) in found.items():
        assert stack == 0 and st == 0 and ld == 0 and regs <= 128, (key, found[key])
