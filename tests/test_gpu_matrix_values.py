"""Matrix literals and properties on the device."""
import pytest

from tests.effects import MATRIX_PROPS, matrix_asset
from tests.helpers import Instance, Lockstep, RefWorld

pytestmark = pytest.mark.gpu


def test_matrix_values_on_the_device(ctx, orc):
    """matCxR literals and properties through every WGSL matrix product (the asset of
    tests/test_host_exec_cpu.py::test_matrix_values_generated_code_equals_interpreter): two instances with different
    property records. Only multiplies and adds in a fixed order under -fmad=false: bit-exact."""
    asset = matrix_asset(4096)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(8192, size // 4, [Instance(0, 4096, alive=0, seed=21), Instance(4096, 4096, alive=0, seed=22)], dt=1 / 20)
    Lockstep(ctx, orc, ref, asset, props=[MATRIX_PROPS, {}]).run([[2000 if f == 0 else 60, 900 if f % 3 == 0 else 0] for f in range(12)])
