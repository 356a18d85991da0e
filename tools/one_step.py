"""One optimizer step of BASELINE config 3 (2 micro-batches of 32, 3x128x128, T=200) between cudaProfilerStart/Stop,
after warm-up steps, for profilers to capture
(ncu --profile-from-start off ...)."""
import sys, io, contextlib, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import cold_diffusion_models_b200 as cdm

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
    gd = cdm.GaussianDiffusion(u, image_size=128, device_of_kernel='cuda', channels=3, timesteps=200, kernel_std=0.01,
                               kernel_size=15, blur_routine='Exponential_reflect', sampling_routine='x0_step_down').cuda()
    tr = cdm.Trainer(gd, None, image_size=128, train_batch_size=B, gradient_accumulate_every=2, results_folder='/tmp/onestep',
                     dataset='synthetic')
xs = [torch.rand(B, 3, 128, 128, device='cuda') * 2 - 1 for _ in range(2)]
for _ in range(2):
    tr.train_step(batches=xs)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
tr.train_step(batches=xs)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
print("done")
