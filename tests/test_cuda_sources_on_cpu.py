"""The library's CUDA-core kernel SOURCES executed on the CPU (tests/simt_cpu: g++ build of the .cu files against a shim
<cuda_runtime.h>, one fiber per CUDA thread) behind the real host code, against the reference goldens.

The host-logic suites (tests/test_*_host_logic.py) normally run on the numpy statement of the C ABI (tests/abi_emulator.py);
with COLDDIFF_ABI_BACKEND=cuda_source the same tests run on the kernels themselves -- every SIMT kernel of the training step,
the degradations, the reverse-process updates, the `Model` training kernels, the optimizer; the tensor-core convolutions are replaced
by the library's own fp32 CUDA-core convolution kernels.  All 28 host-logic tests pass that way (about 13 minutes):

    COLDDIFF_ABI_BACKEND=cuda_source python -m pytest tests/test_unet_host_logic.py tests/test_model2_host_logic.py \\
        tests/test_packages_host_logic.py

This module runs a representative subset of them (about a minute) in every CPU test run; the rest on demand with the command above."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

SUBSET = [
    'test_unet_host_logic.py::test_unet_forward_and_every_gradient_on_the_emulated_abi',      # ConvNeXt Unet forward + backward kernels
    'test_unet_host_logic.py::test_trainer_step_equals_torch_adam_and_ema_on_the_emulated_abi',   # blur q_sample, loss, fused Adam + EMA
    'test_model2_host_logic.py::test_inference_forward_and_sampling_on_the_emulated_abi',     # GroupNorm / softmax attention / step-down
    'test_packages_host_logic.py::test_device_resident_dataset_matches_the_torchvision_pipeline',
]


def test_host_logic_subset_on_the_cuda_kernel_sources():
    env = dict(os.environ, COLDDIFF_ABI_BACKEND='cuda_source')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-x', '-q', '-p', 'no:cacheprovider'] + [os.path.join(HERE, n) for n in SUBSET],
                       env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1500:]
    assert ('%d passed' % len(SUBSET)) in r.stdout, r.stdout[-500:]
