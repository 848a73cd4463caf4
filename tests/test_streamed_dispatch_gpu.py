"""GPU: the zonal spectrum and the conservative regridder (`_streamed.place`)
on CUDA tensors, for each case of tests/test_streamed_dispatch_cpu.py.

Inputs that torch is still producing behind tens of milliseconds of queued
work are read only once produced, the time-sum accumulator is zeroed before
the entry adds into it, and a result read right after the call is complete.
The operators do not wait on the host: the context orders its stream after
torch's current stream and that stream after its own.  Each result is a CUDA
tensor bit-equal to the result of the `_host` entry on the NumPy input."""
import numpy as np
import pytest

from test_streamed_dispatch_cpu import PLACED
from weatherbench2_b200 import xarray_lite as xl

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
  pytest.skip('needs a CUDA device', allow_module_level=True)


def _values(r):
  return r.data if isinstance(r, xl.DataArray) else r


@pytest.mark.parametrize('case', PLACED)
def test_inputs_still_being_produced_are_ordered(case):
  make, _, shape = PLACED[case]
  x = np.random.RandomState(1).standard_normal(shape).astype(np.float32)
  want = _values(make(x)())
  gen = torch.Generator(device='cuda')
  gen.manual_seed(0)
  ballast = torch.randn((8192, 8192), device='cuda', generator=gen)
  dx = torch.from_numpy(x).cuda()
  torch.cuda.synchronize()
  y = ballast
  for _ in range(6):  # ~tens of ms of queued work ahead of the input
    y = y @ ballast
    y = y / y.abs().max()
  got = _values(make(dx + y[0, 0] * 0.0)())  # no sync
  assert isinstance(got, torch.Tensor) and got.is_cuda
  np.testing.assert_array_equal(got.cpu().numpy(), want)
