"""The contents checks of the engine wrappers on CUDA tensors: each bad-contents case of test_engine_checks_cpu.py,
which stops at the device check on CPU tensors, raises its own QRecError once its tensors are on the device.
Needs a GPU."""
import pytest

from test_engine_checks_cpu import CASES, check_cases

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('cases', CASES, ids=[f.__name__ for f in CASES])
def test_contents_checks_on_cuda_tensors(cases):
    import torch
    assert torch.cuda.is_available()
    check_cases(cases(torch, 'cuda'), on_device=True)
