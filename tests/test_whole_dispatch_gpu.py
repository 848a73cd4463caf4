"""GPU: the device-only operators (`_streamed.run_whole`) on CUDA tensors, for
each family of tests/test_whole_dispatch_cpu.py.

  * Inputs that torch is still producing behind tens of milliseconds of queued
    work are read only once produced, and a result read with `.cpu()` right
    after the call is complete.  The operators do not wait on the host: the
    context orders its stream after torch's current stream and that stream
    after its own.
  * A mix of NumPy and CUDA operands, with the first operand on either side,
    runs on the device and gives the all-NumPy result."""
import numpy as np
import pytest

from test_whole_dispatch_cpu import FAMILIES, _numpy

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
  pytest.skip('needs a CUDA device', allow_module_level=True)

NTIME = 4


@pytest.fixture(scope='module')
def ballast():
  gen = torch.Generator(device='cuda')
  gen.manual_seed(0)
  return torch.randn((8192, 8192), device='cuda', generator=gen)


@pytest.mark.parametrize('family', FAMILIES)
def test_inputs_still_being_produced_are_ordered(family, ballast):
  make = FAMILIES[family][2]
  want = make(NTIME, _numpy)()
  uploaded = {}

  def upload(name, a):
    uploaded[name] = torch.from_numpy(a).cuda()
    return a

  make(NTIME, upload)
  torch.cuda.synchronize()
  y = ballast
  for _ in range(6):  # ~tens of ms of queued work ahead of the inputs
    y = y @ ballast
    y = y / y.abs().max()
  zero = y[0, 0] * 0.0
  got = make(NTIME, lambda name, a: uploaded[name] + zero)()  # no sync
  assert got.is_cuda
  np.testing.assert_array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize('first_on_device', [False, True])
@pytest.mark.parametrize('family', [f for f, (_, operands, _) in
                                    FAMILIES.items() if len(operands) > 1])
def test_mixed_residency_runs_on_the_device(family, first_on_device):
  _, operands, make = FAMILIES[family]
  want = make(NTIME, _numpy)()

  def wrap(name, a):
    if (name == operands[0]) == first_on_device:
      return torch.from_numpy(a).cuda()
    return a

  got = make(NTIME, wrap)()
  assert isinstance(got, torch.Tensor) and got.is_cuda
  np.testing.assert_array_equal(got.cpu().numpy(), want)
