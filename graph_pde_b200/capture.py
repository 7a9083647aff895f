"""CUDA-graph replay of a whole model forward (SURVEY 8(f2)).

The small-graph regimes of the reference -- the MGKN V-cycle (13 NNConv calls per depth iteration on a few
thousand nodes, neurips1_MGKN.py:72-84) and config 1 -- are launch bound: one forward is ~150 kernel launches of
a few microseconds each.  Everything this library launches is capture-safe once the per-graph plan and the
per-parameter snapshots exist (plan creation synchronises, so it must happen in the warm-up): buffers come from
the torch caching allocator, tensor maps are encoded on the host, no call synchronises the device.

    g = GraphedForward(model, data)        # warm-up (builds plans / edge features), then capture
    data.x.copy_(new_x)                    # inputs are STATIC tensors: refresh them in place
    out = g.replay()                       # same tensor object every time

Inference only (the autograd graph is not captured); parameters and edge attributes must not change between
replays -- re-create the object after an optimiser step or a new mesh."""
import torch


class GraphedForward(object):
    def __init__(self, model, *inputs, warmup=3):
        if not torch.cuda.is_available():
            raise RuntimeError('GraphedForward needs a CUDA device')
        self.model = model
        self.inputs = inputs
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.no_grad(), torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                model(*inputs)
        torch.cuda.current_stream().wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.output = model(*inputs)

    def replay(self):
        self.graph.replay()
        return self.output

    __call__ = replay
