"""`get_model(args, with_time_emb=True)` of snowification/diffusion/model/get_model.py:4-38: the network by `args.model`
('UnetConvNext' | 'UnetResNet') and, for the ResNet family, by `args.dataset` ('cifar10*' -> 32x32, 'celebA*' -> 128x128)."""
from ...unet import Unet
from ...model2 import Model


def get_model(args, with_time_emb=True):
    if args.model == 'UnetConvNext':
        return Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3, with_time_emb=with_time_emb, residual=False)
    if args.model == 'UnetResNet':
        # with_time_emb=False: the drivers' one-shot model (train.py / test.py build it for every run); it keeps the
        # time-embedding layers and runs them at t = 0 when called without t (unet_resnet.py:291-301)
        for name, res in (('cifar10', 32), ('celebA', 128)):
            if name in args.dataset:
                return Model(resolution=res, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2,
                             attn_resolutions=(16,), dropout=0.1, with_time_emb=with_time_emb)
    return None
