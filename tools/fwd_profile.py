"""One no_grad Unet forward (config 3 network, batch 32) between cudaProfilerStart/Stop after warm-up: the command behind the
`ncu --profile-from-start off --set full -k regex:...` captures of the forward kernels."""
import sys, io, contextlib, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import cold_diffusion_models_b200 as cdm

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
x = torch.rand(B, 3, 128, 128, device='cuda') * 2 - 1
t = torch.randint(0, 200, (B,), device='cuda')
with torch.no_grad():
    for _ in range(2):
        u(x, t)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    u(x, t)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStop()
print("done")
