"""GraphedTrainStep: a whole training step (forward, loss, backward, optimizer.step()) replayed from one CUDA graph
against the same steps taken eagerly, on two copies of a model with identical parameters and Adam(capturable=True).
pytest -m gpu."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.helpers import GOLDEN, ei64, rel_err, t

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
# eager against replayed: the same kernels, only the order of the fp32 atomic additions differs (f16 rounds what
# those sums feed into, so an ulp flip of a 16-bit value shows at its precision)
TOL = {'f16x2': 1e-4, 'fp32': 1e-4, 'f16': 3e-3, 'bf16': 3e-3}


class _Data(object):
    pass


def _cfg1_data(seed=0):
    g = np.load(os.path.join(GOLDEN, 'g2_cfg1_ball16.npz'))
    d = _Data()
    d.x, d.edge_index, d.edge_attr = t(g['node_x']).to(DEV), ei64(g['edge_index']).to(DEV), t(g['edge_attr']).to(DEV)
    gen = torch.Generator().manual_seed(seed)
    y = torch.randn(d.x.size(0), 1, generator=gen).to(DEV)
    return d, y


def _clone_data(d):
    c = _Data()
    c.x, c.edge_index, c.edge_attr = d.x.clone(), d.edge_index.clone(), d.edge_attr.clone()
    return c


def _kernelnn(precision, width=32, depth=3):
    from graph_pde_b200.models import KernelNN
    torch.manual_seed(0)
    return KernelNN(width, 64, depth, 6, in_width=6, precision=precision).to(DEV)


def _pair(factory):
    a, b = factory(), factory()
    b.load_state_dict(a.state_dict())
    return a, b


def _adam(model):
    return torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True)


def _kernelnn_loss(model):
    return lambda d, y: F.mse_loss(model(d).view(-1), y.view(-1))


def _eager_step(loss_fn, opt, *inputs):
    opt.zero_grad(set_to_none=True)
    loss = loss_fn(*inputs)
    loss.backward()
    opt.step()
    return loss.detach()


def _assert_same(loss_g, loss_e, model_g, model_e, tol, what, params=True, grads=False):
    """Loss, (``params``) the parameters after the optimizer step and (``grads``) the gradients agree within ``tol``."""
    assert rel_err(loss_g, loss_e) < tol, (what, float(loss_g), float(loss_e))
    for (name, pg), pe in zip(model_g.named_parameters(), model_e.parameters()):
        if grads:
            err = rel_err(pg.grad, pe.grad)
            assert err < tol, (what, name, 'grad', err)
        if params:
            err = rel_err(pg, pe)
            assert err < tol, (what, name, err)


@pytest.mark.parametrize('precision,width', [('f16x2', 32), ('f16', 32), ('fp32', 32), ('f16x2', 64), ('f16', 64)])
def test_replay_equals_eager_kernelnn(precision, width, edge_kernel_mode):
    """Width 32 trains through the CUDA-core backward, width 64 through the tensor-core backward.  The tensor-core
    backward at f16 rounds its gradients to 16 bits, so a gradient entry near zero can take either sign in two runs of
    the same step, eager or replayed; Adam's first steps move every entry by about lr whatever its size, which turns
    such a sign into a difference of 2 lr.  There only the losses and the first step's gradients are compared."""
    from graph_pde_b200 import GraphedTrainStep
    model_e, model_g = _pair(lambda: _kernelnn(precision, width))
    opt_e, opt_g = _adam(model_e), _adam(model_g)
    d, y = _cfg1_data()
    dg, yg = _clone_data(d), y.clone()
    step = GraphedTrainStep(_kernelnn_loss(model_g), model_g, opt_g, dg, yg)
    for i in range(5):
        loss_e = _eager_step(_kernelnn_loss(model_e), opt_e, d, y)
        loss_g = step.replay()
        _assert_same(loss_g, loss_e, model_g, model_e, TOL[precision], 'step %d' % i,
                     params=(precision, width) != ('f16', 64), grads=i == 0)


def test_new_samples_are_picked_up():
    from graph_pde_b200 import GraphedTrainStep
    model_e, model_g = _pair(lambda: _kernelnn('f16x2'))
    opt_e, opt_g = _adam(model_e), _adam(model_g)
    d, y = _cfg1_data()
    dg, yg = _clone_data(d), y.clone()
    step = GraphedTrainStep(_kernelnn_loss(model_g), model_g, opt_g, dg, yg)
    first = float(step.replay())
    _eager_step(_kernelnn_loss(model_e), opt_e, d, y)
    gen = torch.Generator().manual_seed(1)
    for i in range(3):
        x2 = torch.randn(d.x.shape, generator=gen).to(DEV)
        ea2 = d.edge_attr + 0.1 * torch.randn(d.edge_attr.shape, generator=gen).to(DEV)
        y2 = torch.randn(y.shape, generator=gen).to(DEV)
        for dst, src in ((dg.x, x2), (dg.edge_attr, ea2), (yg, y2)):
            dst.copy_(src)
        d.x, d.edge_attr, y = x2.clone(), ea2.clone(), y2.clone()
        loss_e = _eager_step(_kernelnn_loss(model_e), opt_e, d, y)
        loss_g = step.replay()
        _assert_same(loss_g, loss_e, model_g, model_e, TOL['f16x2'], 'sample %d' % i)
        assert abs(float(loss_g) - first) > 1e-3 * abs(first)


def _burgers():
    from graph_pde_b200.models import MGKN
    g = np.load(os.path.join(GOLDEN, 'g5_mgkn_burgers1d.npz'))

    def factory():
        torch.manual_seed(0)
        return MGKN(width=32, ker_width=64, depth=2, ker_in=4, in_width=2, s=int(g['s'])).to(DEV)
    n = int(g['n_edge_sets'])
    X = [t(g['X/%d' % l]).to(DEV) for l in range(int(g['n_levels']))]
    eis = [ei64(g['edge_index/%d' % i]).to(DEV) for i in range(n)]
    eas = [t(g['edge_attr/%d' % i]).to(DEV) for i in range(n)]
    y = torch.randn(X[0].size(0), 1, generator=torch.Generator().manual_seed(0)).to(DEV)
    return factory, (X, None, eis, eas), y


def test_formulation_b_is_captured_mgkn_burgers(edge_kernel_mode):
    """The orthogonal Burgers MGKN: small graphs whose convs run the per-edge kernel matrices under 'auto'."""
    from graph_pde_b200 import GraphedTrainStep
    from graph_pde_b200.nn_conv import stats
    factory, data, y = _burgers()
    model_e, model_g = _pair(factory)
    opt_e, opt_g = _adam(model_e), _adam(model_g)
    loss_of = lambda m: (lambda data, y: F.mse_loss(m(data).view(-1), y.view(-1)))     # noqa: E731
    data_g = ([x.clone() for x in data[0]], None, [e.clone() for e in data[2]], [a.clone() for a in data[3]])
    yg = y.clone()

    k0 = stats.get('edge_kernel_passes', 0)
    loss_e = _eager_step(loss_of(model_e), opt_e, data, y)
    per_step = stats.get('edge_kernel_passes', 0) - k0
    assert (per_step > 0) == (edge_kernel_mode == 'auto'), per_step
    k0 = stats.get('edge_kernel_passes', 0)
    step = GraphedTrainStep(loss_of(model_g), model_g, opt_g, data_g, yg, warmup=1)
    assert stats.get('edge_kernel_passes', 0) - k0 == 2 * per_step       # one warm-up step, then the captured one
    for i in range(3):
        if i:
            loss_e = _eager_step(loss_of(model_e), opt_e, data, y)
        k0 = stats.get('edge_kernel_passes', 0)
        loss_g = step.replay()
        assert stats.get('edge_kernel_passes', 0) == k0                  # a replay runs none of the Python sequencing
        _assert_same(loss_g, loss_e, model_g, model_e, TOL['f16'], 'step %d' % i, grads=i == 0)


def _snapshot(model, opt):
    return ([p.detach().clone() for p in model.parameters()],
            {id(p): {k: v.clone() if torch.is_tensor(v) else v for k, v in s.items()} for p, s in opt.state.items()})


def test_construction_changes_nothing():
    from graph_pde_b200 import GraphedTrainStep
    d, y = _cfg1_data()
    # a fresh optimizer: the state the warm-up created is reset to Adam's initial zeros
    model = _kernelnn('f16')
    opt = _adam(model)
    params, _ = _snapshot(model, opt)
    GraphedTrainStep(_kernelnn_loss(model), model, opt, d, y)
    assert all(torch.equal(a, b) for a, b in zip(params, model.parameters()))
    assert opt.state and all(not v.any() for s in opt.state.values() for v in s.values() if torch.is_tensor(v))
    # an optimizer with state
    for _ in range(2):
        _eager_step(_kernelnn_loss(model), opt, d, y)
    params, state = _snapshot(model, opt)
    GraphedTrainStep(_kernelnn_loss(model), model, opt, d, y)
    assert all(torch.equal(a, b) for a, b in zip(params, model.parameters()))
    for p, s in opt.state.items():
        assert set(s) == set(state[id(p)])
        for k, v in s.items():
            assert torch.equal(v, state[id(p)][k]) if torch.is_tensor(v) else v == state[id(p)][k]


def test_caches_are_refreshed_after_replay():
    from graph_pde_b200 import GraphedTrainStep
    model = _kernelnn('fp32')
    d, y = _cfg1_data()
    step = GraphedTrainStep(_kernelnn_loss(model), model, _adam(model), d, y)
    for _ in range(3):
        step.replay()
    fresh = _kernelnn('fp32')
    fresh.load_state_dict(model.state_dict())
    with torch.no_grad():
        ref = fresh(d)
        assert rel_err(model(d), ref) < 1e-5          # no mode change in between: only the replay's invalidation
        model.eval()
        assert rel_err(model(d), ref) < 1e-5


def test_overflow_is_reported_from_inside_the_graph():
    from graph_pde_b200 import GraphedTrainStep
    d, y = _cfg1_data()
    model = _kernelnn('f16')
    step = GraphedTrainStep(_kernelnn_loss(model), model, _adam(model), d, y)
    step.replay()
    rounds = 0
    with pytest.raises(FloatingPointError, match='edge-MLP activations left the fp16 range'):
        for rounds in range(1, 9):
            for lin in (model.conv1.nn.layers[0], model.conv1.nn.layers[2]):
                lin.weight.data.mul_(16.0)
            step.replay()
    assert rounds >= 1
    # the same scaling at bf16, whose range holds it
    model_bf = _kernelnn('bf16')
    step_bf = GraphedTrainStep(_kernelnn_loss(model_bf), model_bf, _adam(model_bf), d, y)
    step_bf.replay()
    for _ in range(rounds):
        for lin in (model_bf.conv1.nn.layers[0], model_bf.conv1.nn.layers[2]):
            lin.weight.data.mul_(16.0)
        step_bf.replay()


def test_kmat_overflow_asks_for_a_new_capture(monkeypatch):
    """A last-layer bias beyond the fp16 range overflows K_e (formulation B) and nothing else.  Eager steps fall back to
    formulation C there; a replayed step reports it, and a new capture falls back like the eager step."""
    from graph_pde_b200 import GraphedTrainStep, nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'on')
    d, y = _cfg1_data()
    model = _kernelnn('f16', depth=1)
    opt = _adam(model)
    step = GraphedTrainStep(_kernelnn_loss(model), model, opt, d, y)
    step.replay()
    good = {k: v.clone() for k, v in model.state_dict().items()}
    model.conv1.nn.layers[4].bias.data.fill_(1e5)
    with pytest.raises(FloatingPointError, match='re-create the GraphedTrainStep'):
        step.replay()
    model.load_state_dict(good)                        # the reported step has been applied: restore, then re-create
    model.conv1.nn.layers[4].bias.data.fill_(1e5)
    opt = _adam(model)
    step = GraphedTrainStep(_kernelnn_loss(model), model, opt, d, y)
    for _ in range(2):
        assert torch.isfinite(step.replay())


def test_refusals():
    from graph_pde_b200 import GraphedTrainStep
    d, y = _cfg1_data()
    model = _kernelnn('f16')
    with pytest.raises(ValueError, match='capturable=True'):
        GraphedTrainStep(_kernelnn_loss(model), model, torch.optim.Adam(model.parameters(), lr=1e-3), d, y)
    with pytest.raises(ValueError, match='capturable=True'):
        GraphedTrainStep(_kernelnn_loss(model), model, torch.optim.SGD(model.parameters(), lr=1e-3), d, y)
    cpu = _kernelnn('f16').cpu()
    with pytest.raises(ValueError, match='CUDA'):
        GraphedTrainStep(_kernelnn_loss(cpu), cpu, _adam(cpu), d, y)


def test_streamed_edge_features_are_refused(monkeypatch):
    from graph_pde_b200 import GraphedTrainStep, nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')
    d, y = _cfg1_data()
    model = _kernelnn('f16')
    model.conv1.edge_feature_bytes = 256 << 10        # a fifth of the 9324 edges' 1.2 MB of h stays resident
    model.conv1.streamed_training = True
    opt = _adam(model)
    params = [p.detach().clone() for p in model.parameters()]
    with pytest.raises(RuntimeError, match='stream'):
        GraphedTrainStep(_kernelnn_loss(model), model, opt, d, y)
    assert all(torch.equal(a, b) for a, b in zip(params, model.parameters()))
