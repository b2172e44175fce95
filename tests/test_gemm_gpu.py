"""GPU parity of yamb_pointwise_gemm (wgmma GEMM) against plain torch fp32 math of the same op:
forward / dgrad / wgrad orientations, operand transforms, BN-statistics and dz epilogues."""
import pytest

from gpu_probe_gemm import CASES, run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(CASES))
def test_gemm_case(built_lib, name):
    assert run_case(name) == 0
