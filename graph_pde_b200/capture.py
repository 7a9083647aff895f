"""CUDA-graph replay of a whole model forward (SURVEY 8(f2)), and of a whole training step.

The small-graph regimes of the reference -- the MGKN V-cycle (13 NNConv calls per depth iteration on a few
thousand nodes, neurips1_MGKN.py:72-84) and config 1 -- are launch bound: one forward is ~150 kernel launches of
a few microseconds each.  Everything this library launches is capture-safe once the per-graph plan and the
per-parameter snapshots exist (plan creation synchronises, so it must happen in the warm-up): buffers come from
the torch caching allocator, tensor maps are encoded on the host, no call synchronises the device.

    g = GraphedForward(model, data)        # warm-up (builds plans / edge features), then capture
    data.x.copy_(new_x)                    # inputs are STATIC tensors: refresh them in place
    out = g.replay()                       # same tensor object every time

GraphedForward is inference only (the autograd graph is not captured); parameters and edge attributes must not change
between replays -- re-create the object after an optimiser step or a new mesh.  GraphedTrainStep captures forward,
loss, backward and the optimiser step together (see its docstring)."""
import torch

from . import nn_conv
from .nn_conv import DiagNNConv, NNConv_old


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


# optimisers whose lazily created state is all zeros (moments and step count), so that "no state yet" can be restored
# by zeroing the state the warm-up created
_ZERO_INIT_OPTIMIZERS = (torch.optim.Adam, torch.optim.AdamW, torch.optim.Adamax)


class GraphedTrainStep(object):
    """One training step -- ``loss_fn(*static_inputs)``, its backward and ``optimizer.step()`` -- replayed from one CUDA
    graph.  On the small fixed meshes of the reference's longest training loops (batch size 1), an eager step waits on
    Python and on host synchronisations rather than on the kernels; a replay launches the whole step at once and
    synchronises once, to read the fp16 overflow counter.

        step = GraphedTrainStep(loss_fn, model, optimizer, data, y)     # optimizer built with capturable=True
        for x, edge_attr, target in samples:                            # every sample on the SAME mesh
            data.x.copy_(x); data.edge_attr.copy_(edge_attr); y.copy_(target)
            loss = step.replay()                                        # the same tensor every time

    ``loss_fn(*static_inputs)`` returns the scalar loss.  The static inputs are read in place: per-sample data goes in by
    ``copy_`` into them.  A new mesh (another edge_index or other shapes) needs a new GraphedTrainStep, and so does a
    change of precision, of the optimiser's hyper-parameters held as Python numbers, or of the model's structure.

    Construction warms the step up on a side stream (this builds the per-mesh plans, whose creation synchronises) and
    then restores the parameters, buffers and optimiser state it found, in place: constructing the object trains
    nothing.  An optimiser with no state yet must be one whose fresh state is zeros (Adam, AdamW, Adamax); take one
    eager step first with any other.  The capture records the weight preparation and the edge-feature pass of every
    NNConv, so every replay recomputes them from the current parameters and edge attributes.  The gradients of the
    captured step live in the graph's memory: do not set them to None between replays.

    After each replay the convs' caches (NNConv_old, NNConv and DiagNNConv) are dropped (the step changed the parameters in place without bumping their
    version counters, so a later eager forward would otherwise use stale prepared weights), and the fp16 range counters
    that the step's edge-feature passes and K_e builds added up on the device are read with one 4-byte copy.  A
    non-zero count raises FloatingPointError.  The optimiser step has been applied by then: restore the parameters
    before going on.  Graphs whose edge features would stream (they do not fit on the device or in the convs' budget)
    are refused: their steps are bound by recomputation, not by launches."""

    def __init__(self, loss_fn, model, optimizer, *static_inputs, warmup=3):
        if not torch.cuda.is_available():
            raise RuntimeError('GraphedTrainStep needs a CUDA device')
        params = list(model.parameters())
        if not params or not all(p.is_cuda for p in params):
            raise ValueError('GraphedTrainStep needs a model whose parameters are all on a CUDA device')
        if not all(g.get('capturable', False) for g in optimizer.param_groups):
            raise ValueError('GraphedTrainStep needs an optimizer built with capturable=True (e.g. '
                             'torch.optim.Adam(params, capturable=True)): only then does optimizer.step() keep its '
                             'step count on the device and run without host synchronisation')
        fresh = [p for g in optimizer.param_groups for p in g['params'] if not optimizer.state.get(p)]
        if fresh and not isinstance(optimizer, _ZERO_INIT_OPTIMIZERS):
            raise ValueError('GraphedTrainStep: %s has no state yet for %d parameters, and its fresh state is not known '
                             'to be zeros: take one eager step before capturing' % (type(optimizer).__name__,
                                                                                     len(fresh)))
        self.loss_fn, self.model, self.optimizer, self.inputs = loss_fn, model, optimizer, static_inputs
        # DiagNNConv keeps no edge features that could stream: only its prepared weights, d and training state
        self._convs = [m for m in model.modules() if isinstance(m, (NNConv_old, DiagNNConv))]
        dev = params[0].device

        # snapshot, warm-up, restore in place
        model_state = [(t, t.detach().clone()) for t in model.state_dict(keep_vars=True).values()
                       if isinstance(t, torch.Tensor)]
        opt_state = {p: {k: v.detach().clone() if torch.is_tensor(v) else v for k, v in s.items()}
                     for p, s in optimizer.state.items() if s}
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                optimizer.zero_grad(set_to_none=True)
                loss_fn(*static_inputs).backward()
                optimizer.step()
        torch.cuda.current_stream(dev).wait_stream(side)
        streamed = any(ef.streamed for c in self._convs if isinstance(c, NNConv_old) for ef in c._h_cache.values())
        with torch.no_grad():
            for t, v in model_state:
                t.copy_(v)
            for p, s in optimizer.state.items():
                old = opt_state.get(p)
                for k, v in s.items():
                    if old is None:
                        if torch.is_tensor(v):
                            v.zero_()
                    elif torch.is_tensor(v) and torch.is_tensor(old.get(k)):
                        v.copy_(old[k])
                    elif k in old:
                        s[k] = old[k]
        self._invalidate()
        if streamed:
            raise RuntimeError('GraphedTrainStep: the edge features of this graph stream (they do not fit on the device '
                               'or in the edge_feature_bytes budget), and streamed edge features are not captured: a '
                               'step over them is bound by their recomputation, not by launches -- train it eagerly')

        # capture one step with every fp16 range counter folded into the sink
        optimizer.zero_grad(set_to_none=True)
        self._sink = nn_conv._CaptureSink(dev)
        self.graph = torch.cuda.CUDAGraph()
        with nn_conv._capturing_into(self._sink), torch.cuda.graph(self.graph):
            loss = loss_fn(*static_inputs)
            loss.backward()
            optimizer.step()
        self.loss = loss.detach()
        self._invalidate()      # capture ran nothing: the caches it filled hold no values

    def _invalidate(self):
        for c in self._convs:
            c.invalidate()
            # the tensor-core backward's state holds its step's autograd graph, and with it the AccumulateGrad nodes of
            # the hidden parameters, which autograd would otherwise reuse on another stream in the next capture
            c._tstate = None

    def replay(self):
        self.graph.replay()
        self._invalidate()
        if nn_conv._OVERFLOW_CHECK:
            self._check_overflow()
        return self.loss

    __call__ = replay

    def _check_overflow(self):
        words = self._sink.words
        n = int(words[0].item())
        if not n:
            return
        n_kmat = int(words[1].item())
        words.zero_()
        if n > n_kmat:
            raise FloatingPointError(
                'graph_pde_b200.GraphedTrainStep: %d blocks of edge-MLP activations left the fp16 range (|h| > 65504 '
                "or NaN) in the replayed step, which has been applied; use precision='bf16' or 'fp32' for this "
                'parameter scale (NNCONV_B200_OVERFLOW_CHECK=0 disables this check and its one host sync per replay)'
                % (n - n_kmat))
        raise FloatingPointError(
            'graph_pde_b200.GraphedTrainStep: %d blocks of the per-edge kernel matrices K_e = W_L h_e + b_L left the '
            'fp16 range in the replayed step, which has been applied (K_e holds the last-layer bias in 16 bits).  An '
            'eager step computes such a graph with the per-source matrices instead, which keep that bias in fp32, and '
            'so does a new capture: restore the parameters and re-create the GraphedTrainStep' % n_kmat)
