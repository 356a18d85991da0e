"""CPU estimate of the TF32-path error of the multi-step GPU parity tests (tests/test_helpers_and_variants_gpu.py): runs the same
calls on CPU tensors through tests/abi_emulator.py with both operands of every tensor-core convolution rounded to TF32 (RN,
like the TFLOAT32 tensor maps), and prints the relative errors against the reference goldens.  Used to set tolerances before a
test first runs on the GPU.  Conservative: single forward of the small net 5.8e-4 here.  Usage: python tools/tf32_estimate.py"""
import os, sys, io, contextlib
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ('', 'tests'):
    sys.path.insert(0, os.path.join(ROOT, p))
import numpy as np, torch
import abi_emulator
abi_emulator.TF32_EMULATION = True
if os.environ.get('COLDDIFF_OPERAND_FORMAT') == 'fp16':      # same estimate with FP16 operands
    abi_emulator._tf32 = lambda a: np.ascontiguousarray(a, dtype=np.float32).astype(np.float16).astype(np.float32)
torch.Tensor.is_cuda = property(lambda self: True)
torch.Tensor.cuda = lambda self, *a, **k: self
import cold_diffusion_models_b200 as cdm
G = os.path.join(ROOT, 'tests', 'golden')
def load(n):
    z=np.load(os.path.join(G,n+'.npz')); return {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}
def rel(a,b): return ((a.double()-b.double()).norm()/(b.double().norm()+1e-30)).item()
def stack(l): return torch.stack([x.detach().float() for x in l])
g=load('unet_small')
with contextlib.redirect_stdout(io.StringIO()):
    u=cdm.Unet(dim=32, dim_mults=(1,2), channels=3)
u.load_state_dict({k[3:]:v for k,v in g.items() if k.startswith('sd:')})
with abi_emulator.patched(), torch.no_grad():
    print('forward', rel(u(g['x'], g['t']), g['y']))
    gf=load('fb_small'); x=gf['x']
    for key in sorted(k[4:] for k in gf if k.startswith('img:')):
        routine, ks, std, T, samp = key.split('|')
        gd=cdm.GaussianDiffusion(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=int(T), kernel_std=float(std), kernel_size=int(ks), blur_routine=routine, sampling_routine=samp)
        for start in (0,1):
            xt,dr,img=gd.sample_from_blur(batch_size=2,img=x,start=start); pre=':%d:'%start+key
            print('sfb', pre, rel(dr,gf['sfb_dr'+pre]), rel(img,gf['sfb_img'+pre]))
        X0s,Xts=gd.all_sample(batch_size=2,img=x)
        print('all', key, rel(stack(X0s),gf['all_X0:'+key]), rel(stack(Xts),gf['all_Xt:'+key]))
    from cold_diffusion_models_b200.resolution_diffusion_pytorch import GaussianDiffusion as RS
    gr=load('resolution_train_small'); x=gr['x']
    for samp in ('x0_step_down','default'):
        gd=RS(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, loss_type='l1', resolution_routine='Incremental_factor_2', train_routine='Final', sampling_routine=samp)
        X0s,Xts=gd.all_sample(batch_size=3,img=x); F_,B_,img=gd.forward_and_backward(batch_size=3,img=x)
        print('res', samp, rel(stack(X0s),gr['all_X0:'+samp]), rel(stack(Xts),gr['all_Xt:'+samp]), rel(stack(B_),gr['fb_B:'+samp]), rel(img,gr['fb_img:'+samp]))
    gd=RS(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, loss_type='l1', resolution_routine='Incremental_factor_2', train_routine='Step', sampling_routine='x0_step_down')
    print('res step loss', abs(gd.p_losses(x, torch.tensor([3,0,2])).item()-gr['loss:Step|l1'].item()))
    gi=load('individual_small'); x=gi['x']
    for samp in ('default','x0_step_down'):
        gd=cdm.GaussianDiffusion(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, kernel_std=0.1, kernel_size=3, blur_routine='Individual_Incremental', sampling_routine=samp)
        xt,dr,img=gd.sample(batch_size=2,img=x)
        print('indiv', samp, abs(gd.p_losses(x,torch.tensor([3,1])).item()-gi['loss'].item()), rel(dr,gi['dr:'+samp]), rel(img,gi['img:'+samp]))
    from cold_diffusion_models_b200.defading_diffusion_pytorch import GaussianDiffusion as DF
    gd_=load('defading_all_small'); x=gd_['x']
    for key in sorted(k[3:] for k in gd_ if k.startswith('x0:')):
        routine,T,samp=key.split('|')
        gd=DF(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=int(T), loss_type='l1', kernel_std=0.6, initial_mask=3, fade_routine=routine, sampling_routine=samp)
        off=(gd_['rx:'+key], gd_['ry:'+key]) if 'Random' in routine else (None,None)
        x0l,xtl=gd.all_sample(batch_size=2, faded_recon_sample=x, _offsets=off)
        print('defade', key, rel(stack(x0l),gd_['x0:'+key]), rel(stack(xtl),gd_['xt:'+key]))
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion as SN
    gs=load('snow_more_small'); x=gs['x']
    for key in sorted(k[5:] for k in gs if k.startswith('fb_F:')):
        fpt,kws,T,samp=key.split('|'); kw={}
        for item in kws.split('-'):
            k,v=item.split('='); kw[k]=(v=='True') if v in ('True','False') else (float(v) if '.' in v else (int(v) if v.isdigit() else v))
        if fpt=='Snow': kw['results_folder']='/tmp'
        with contextlib.redirect_stdout(io.StringIO()):
            gd=SN(u, image_size=(32,32) if fpt=='Snow' else 32, device_of_kernel='cpu', channels=3, timesteps=int(T), loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, **kw)
        if fpt=='Decolorization':
            X0,Xt,_,_=gd.all_sample(batch_size=3,img=x); print('snow all', key[:30], rel(stack(X0),gs['all_X0:'+key]), rel(stack(Xt),gs['all_Xt:'+key]))
        F_,B_,img=gd.forward_and_backward(batch_size=3,img=x); print('snow fb', key[:30], rel(stack(B_),gs['fb_B:'+key]), rel(img,gs['fb_img:'+key]))
    go=load('unet_options_small')
    base={k[3:]:v for k,v in g.items() if k.startswith('sd:')}
    for tag,kw in (('residual',dict(residual=True)),('notime',dict(with_time_emb=False)),('outdim',dict(out_dim=5))):
        with contextlib.redirect_stdout(io.StringIO()):
            uu=cdm.Unet(dim=32, dim_mults=(1,2), channels=3, **kw)
        pre=tag+':sd:'; extra={k[len(pre):]:v for k,v in go.items() if k.startswith(pre)}
        uu.load_state_dict({k: extra.get(k, base.get(k)) for k in uu.state_dict()})
        print('options', tag, rel(uu(go['x'], go['t']), go[tag+':y']))
