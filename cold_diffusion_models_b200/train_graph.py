"""CUDA-graph replay of a training step's forward + backward (`Trainer.enable_cuda_graph`).

One graph holds the A micro-batches of one optimizer step: each one's t / noise draws, degradation, network forward, loss and
engine backward (accumulating into the flat gradient buffer), and the sum of their losses.  Around each replay stay eager: the
batch copy into the graph's static inputs, the weight repacks after an optimizer step, the host-side random draws, the fused
Adam + EMA step and the gradient zeroing.

Host-side random draws cannot happen inside a graph.  While a step is warmed up or captured, `recording()` returns the step's
HostDraws, and the code that would draw on the host registers a device slot there instead: the `Model`'s dropout seeds
(model2_train._res_fwd) and the snow layers of `random_snow` (snowification.GaussianDiffusion.p_losses).  Before every replay
`HostDraws.stage()` makes the same draws, from the same generators, in the order the eager step makes them, and writes them
where the captured kernels read them.  The torch CUDA generator needs no staging: its draws inside a graph advance its offset
at every replay (graph-safe Philox), as the eager launches would.
"""
import numpy as np
import torch

from . import graphs

_RECORDING = None


def recording():
    """the HostDraws of the training step being warmed up or captured; None while launches are eager"""
    return _RECORDING


class HostDraws:
    """the host-side draws of one captured step, in eager order, and the device memory the graph reads them from"""

    def __init__(self, device):
        self.device = device
        self.seeds = torch.zeros(0, dtype=torch.int64, device=device)
        self.bufs = []
        self.reset()

    def reset(self):
        """start the schedule again: the capture repeats the warm-up's requests and gets the same slots and buffers back"""
        self.order, self.nseeds, self.nbufs = [], 0, 0

    def dropout_seed(self):
        """-> 1-element int64 device view that holds, at every replay, the seed the eager forward draws here on the host"""
        k = self.nseeds
        self.nseeds += 1
        if k >= self.seeds.numel():         # only during the warm-up: the views handed out before stay unused
            self.seeds = torch.zeros(max(64, 2 * (k + 1)), dtype=torch.int64, device=self.device)
        self.order.append(k)
        return self.seeds[k:k + 1]

    def host_call(self, fn):
        """fn() runs before every replay, at its place in the order of the draws"""
        self.order.append(fn)

    def buffer(self, shape, init=None, dtype=torch.float32):
        """a device tensor that lives as long as the graph (allocated by the warm-up; the capture gets the same one back)"""
        k = self.nbufs
        self.nbufs += 1
        if k == len(self.bufs):
            b = torch.zeros(shape, dtype=dtype, device=self.device)
            if init is not None:
                b.copy_(init)
            self.bufs.append(b)
        return self.bufs[k]

    def stage(self):
        seeds = []
        for item in self.order:
            if callable(item):
                item()
            else:   # the draw of model2_train._res_fwd's eager path
                seeds.append(int(torch.randint(0, 2 ** 62, (1,)).item()))
        if seeds:
            # pageable source: CUDA stages it before the call returns, so the temporary may go at once
            self.seeds[:len(seeds)].copy_(torch.tensor(seeds, dtype=torch.int64), non_blocking=True)


class StepGraph:
    def __init__(self, graph, statics, draws, loss):
        self.graph, self.statics, self.draws, self.loss = graph, statics, draws, loss

    def replay(self, ds):
        for st, d in zip(self.statics, ds):
            if isinstance(st, tuple):
                for s, x in zip(st, d):
                    s.copy_(x, non_blocking=True)
            else:
                st.copy_(d, non_blocking=True)
        self.draws.stage()
        self.graph.replay()
        return self.loss


def capture(trainer, ds):
    """warm up and capture trainer._accumulate over static copies of the micro-batches `ds`.  The warm-up runs the step once
    for real (it allocates every workspace and attaches the gradient views); the flat gradient and every random generator
    the step reads are put back as they were, so the next replay computes what the next eager step would."""
    global _RECORDING
    eng = trainer._unet.engine
    dev = eng.flat_grad.device
    own = lambda x: x.to(dev, copy=True).contiguous()
    statics = [tuple(own(x) for x in d) if isinstance(d, (tuple, list)) else own(d) for d in ds]
    eng.prepare_training_weights()
    grad0 = eng.flat_grad.clone()
    rng = (torch.cuda.get_rng_state(dev), torch.get_rng_state(), np.random.get_state())
    draws = HostDraws(dev)

    def step():
        draws.reset()
        return trainer._accumulate(statics)[0]
    try:
        _RECORDING = draws
        graph, loss = graphs.capture(step, dev)
    finally:
        _RECORDING = None
    eng.flat_grad.copy_(grad0)
    torch.cuda.set_rng_state(rng[0], dev)
    torch.set_rng_state(rng[1])
    np.random.set_state(rng[2])
    return StepGraph(graph, statics, draws, loss)
