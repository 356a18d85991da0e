"""CUDA-graph capture and replay: the inference forward of `Unet` and `Model` (`engine.enable_cuda_graph`; a sampling loop calls
R(x_t, t) T times with identical shapes, and one graph launch replaces the ~150-200 launches of the Python schedule) and the
training step (`Trainer.enable_cuda_graph`, train_graph.py).

A graph holds the addresses it was captured with.  The packed weight operands are refilled in place, so a graph follows
in-place weight updates (optimizer steps, load_state_dict) without a new capture; a parameter whose storage moved
(flatten_params, load_state_dict(assign=True), `p.data = ...`) is seen by its address, and every graph is captured again."""
import torch

_CAPTURE_STREAMS = {}


def capture_stream(device):
    """the one stream per device on which every graph is warmed up and captured.  The split GroupNorm (planes above 128²)
    keeps its partials in a buffer cached per (device, stream) that cannot grow during a capture: the warm-up on this same
    stream grows it to the shape first."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    s = _CAPTURE_STREAMS.get(idx)
    if s is None:
        s = _CAPTURE_STREAMS[idx] = torch.cuda.Stream(device=idx)
    return s


def capture(fn, device):
    """-> (graph, what fn() returned inside the capture).  fn runs once outside the capture first (the warm-up allocates every
    workspace), both on the device's capture stream, ordered after the work already queued on the current stream."""
    cs = capture_stream(device)
    cs.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cs):
        fn()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cs):
        out = fn()
    torch.cuda.current_stream().wait_stream(cs)
    return graph, out


class GraphCache(dict):
    """captured graphs by key, all captured with the same addresses `ptrs`"""
    ptrs = None

    def lookup(self, key, ptrs, make):
        """the graph of `key`, made by make() when missing; every graph is dropped first when `ptrs` changed"""
        if ptrs != self.ptrs:
            self.clear()
            self.ptrs = ptrs
        g = self.get(key)
        if g is None:
            g = self[key] = make()
        return g


class GraphedForward:
    """the inference forward of UnetEngine and ModelEngine, replayed from one graph per input shape (B, C, H, W) with static x
    and t.  The engine calls _init_graphs(module, forward, prepare): `module` is the network, whose parameters' addresses the
    graphs hold; forward(x, t) launches the forward to capture; prepare(params) refills the packed operands when a parameter
    changed, and the engine's mark_weights_dirty() makes them all stale.  The switch is stored on the network (`_cuda_graph`),
    so _apply and a deep copy (the Trainer's EMA model) keep it; the graphs are per engine."""

    def _init_graphs(self, module, forward, prepare):
        self._graph_net, self._graph_forward, self._graph_prepare = module, forward, prepare
        self.drop_graphs()

    @property
    def use_cuda_graph(self):
        return getattr(self._graph_net, '_cuda_graph', False)

    def enable_cuda_graph(self, flag=True):
        self._graph_net._cuda_graph = bool(flag)
        self.drop_graphs()

    def drop_graphs(self):
        """forget every captured graph: parameter storage or workspaces moved, and the graphs hold their old addresses"""
        self._graphs, self._graph_params = GraphCache(), None

    def forward_graphed(self, x, t):
        """the inference forward, replayed from one graph per input shape (B, C, H, W); returns a clone of the graph's output"""
        # the parameter list is cached (walks of the module tree were most of a replay's host time); load_state_dict sets it
        # to None, as it may replace the Parameter objects (assign=True)
        if self._graph_params is None:
            self._graph_params = list(self._graph_net.parameters())
        ptrs = tuple(p.data_ptr() for p in self._graph_params)
        if ptrs != self._graphs.ptrs:
            self.mark_weights_dirty()       # new storage has its own version counter: repack whatever the versions say
        # the packs refill persistent tensors, so a graph stays valid across weight updates: repack before every replay
        # (a no-op when no parameter changed)
        self._graph_prepare(self._graph_params)
        graph, sx, st, so = self._graphs.lookup(tuple(x.shape), ptrs, lambda: self._capture(x, t))
        sx.copy_(x)
        st.copy_(t)
        graph.replay()
        return so.clone()

    def _capture(self, x, t):
        sx = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        sx.copy_(x)
        st = torch.empty((x.shape[0],), device=x.device, dtype=torch.int64)
        st.copy_(t)
        graph, so = capture(lambda: self._graph_forward(sx, st), x.device)
        return graph, sx, st, so
