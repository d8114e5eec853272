"""The GEMM kernels of the product library fit Hopper's register file: ptxas keeps every wgmma in flight (no serialization
note for any kernel) and the bf16-mode GEMM mainloops never spill.  Reads the ptxas -v log of the build; no GPU needed."""
import os

import pytest

from scalerl_b200 import build as B

PRODUCT = set(B.SOURCES)
# bf16-mode (SPLIT = 0) instantiations of the resident-window conv kernels and the TMA implicit-GEMM kernel
GEMM_KERNELS = ('14res_fwd_kernel', '16res_wgrad_kernel', '16igemm_tma_kernel')


@pytest.fixture(scope='module')
def report():
    path = os.path.join(B.HERE, 'build', 'ptxas.log')
    if not os.path.exists(path):
        B.build(force=True)
    rep = B.ptxas_report(path)
    assert PRODUCT <= set(rep), f'ptxas log lacks sources {sorted(PRODUCT - set(rep))}'
    return rep


def test_no_serialized_wgmma(report):
    bad = {k: v['serialized'] for src in PRODUCT for k, v in report[src].items() if v['serialized']}
    assert not bad, f'wgmma serialized by ptxas: {bad}'


def test_bf16_gemm_kernels_do_not_spill(report):
    kernels = {k: v for src in PRODUCT for k, v in report[src].items()
               if any(n in k for n in GEMM_KERNELS) and 'ELi0EEEv' in k}
    assert len(kernels) >= 12, sorted(kernels)          # 6 res_fwd, 3 res_wgrad, >= 3 igemm_tma problems
    spills = {k: (v['spill_stores'], v['spill_loads']) for k, v in kernels.items() if v['spill_stores'] or v['spill_loads']}
    assert not spills, f'spilling GEMM kernels (bytes stored, loaded): {spills}'
