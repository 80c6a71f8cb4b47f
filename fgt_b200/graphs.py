"""Host caches of the network modules (NativeNet: packed weights, workspaces, CUDA graphs) and CUDA-graph replay of
a whole model forward (opt-in).

Every forward here is a fixed sequence of kernel launches over cached workspaces, so after one eager
call per input geometry the sequence is captured into a CUDA graph and replayed: one graph launch
instead of 30-300 ctypes launches (LAFC and RAFT are host-launch bound otherwise; FGT is GPU bound and
gains little). TMA descriptors are encoded on the host at capture time and baked into the graph, which
is valid because all buffers are static. Inputs are copied into static tensors, outputs are cloned.
"""
import torch
import torch.nn as nn

from . import lib


class GraphedCall:
    def __init__(self, fn):
        self.fn = fn
        self.entries = {}

    def __call__(self, *tensors):
        key = tuple((tuple(t.shape), t.dtype, t.device.index) for t in tensors)
        e = self.entries.get(key)
        if e is None:
            self.entries[key] = {}
            return self.fn(*tensors)  # eager: packs weights, allocates workspaces, sets kernel attributes
        if "graph" not in e:
            e["inp"] = [t.clone() for t in tensors]
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            l0 = lib.COUNTERS["launches"]
            with torch.cuda.graph(g):
                e["out"] = self.fn(*e["inp"])
            e["launches"] = lib.COUNTERS["launches"] - l0
            e["graph"] = g
        for s, t in zip(e["inp"], tensors):
            s.copy_(t, non_blocking=True)
        e["graph"].replay()
        lib.COUNTERS["launches"] += e["launches"]
        out = e["out"]
        if isinstance(out, torch.Tensor):
            return out.clone()
        return type(out)(o.clone() if isinstance(o, torch.Tensor) else o for o in out)


def workspace(bufs, name, shape, dev, dtype=torch.float32, zero=False):
    """Buffer `name` of the workspace dict `bufs`, allocated on first use: bfloat16 as lib.empty_split, else [*shape]."""
    if name not in bufs:
        t = lib.empty_split(shape, dev) if dtype == torch.bfloat16 else torch.empty(shape, dtype=dtype, device=dev)
        bufs[name] = t.zero_() if zero else t
    return bufs[name]


def _drop_weights(net, incompatible_keys):
    net._packed = {}
    net._drop_graphs()


class NativeNet(nn.Module):
    """Host caches of a network whose forward runs on the native kernels: packed weights per precision (`_packed`),
    workspaces per input geometry (`_geo`) and, while enabled, CUDA graphs per call (`_graphs`, keyed by the call's
    non-tensor arguments). Packed weights are copies of the parameters and graphs hold the addresses of packed weights
    and workspaces, so `.to()` / `.half()` / ... drop all three, and a state-dict load drops the packed weights and the
    graphs, also when the load is called on a wrapper module or on nn.DataParallel."""

    def __init__(self):
        super().__init__()
        self._packed = {}
        self._geo = {}
        self._graphs = None
        self.register_load_state_dict_post_hook(_drop_weights)

    def _drop_graphs(self):
        if self._graphs:
            self._graphs.clear()

    def _apply(self, fn, *a, **k):
        self._packed = {}
        self._geo = {}
        self._drop_graphs()
        return super()._apply(fn, *a, **k)

    def _allocators(self, key, dev, mixed):
        """(B, A) workspace allocators of geometry `key`: B(name, shape, dtype=fp32) and A(name, shape) for the 16-bit
        activations of the path, split-bf16 (fp32 path) or fp16 (mixed)."""
        bufs = self._geo.setdefault(key, {})
        return ((lambda nm, s, dtype=torch.float32: workspace(bufs, nm, s, dev, dtype)),
                (lambda nm, s, zero=False: workspace(bufs, nm, s, dev, lib.act16_dtype(mixed), zero)))

    def enable_cuda_graph(self, on=True):
        """Replay whole forwards as CUDA graphs, one per input geometry and call key."""
        self._graphs = {} if on else None

    def _graphed(self, key, fn, *tensors):
        """fn(*tensors) through the GraphedCall of `key` (the call's non-tensor arguments)."""
        gc = self._graphs.get(key)
        if gc is None:
            gc = self._graphs[key] = GraphedCall(fn)
        return gc(*tensors)
