"""Callers of the NNConv hot path, with the module signatures and state-dict layouts of the reference
scripts so that their checkpoints / training loops carry over:

* ``DenseNet``      -- graph-neural-operator/utilities.py:201-227 (parameter container of the edge MLP)
* ``KernelNN``      -- graph-neural-operator/UAI1_full_resolution.py:14-33 (variants UAI7_evaluate.py:26-35:
                       no ReLU after the last conv -> ``relu_last=False``)
* ``KernelInduced`` -- multipole-graph-neural-operator/neurips1_MGKN.py:20-89   (MGKN V-cycle)
* ``MKGN``          -- multipole-graph-neural-operator/MGKN_general_darcy2d.py:21-94 (mid conv with root,
                       level-sliced node ranges)
* ``MGKN``          -- multipole-graph-neural-operator/MGKN_orthogonal_burgers1d.py:21-86

Only the conv applications run in the CUDA library; the pointwise lifts / projections (fc*) stay
torch.nn.Linear exactly as in the reference (they are not on the hot path, SURVEY 8(a)).
"""
import os

import numpy as np
import torch
import torch.nn.functional as F

from .nn_conv import NNConv, NNConv_old

# NNCONV_B200_FUSED_STEPS=0: KernelInduced inference runs the reference's op sequence (conv, add, ReLU as separate kernels)
_FUSED_STEPS = os.environ.get('NNCONV_B200_FUSED_STEPS', '1') != '0'


class DenseNet(torch.nn.Module):
    """Linear -> nonlinearity -> ... -> Linear; ``self.layers`` is a ModuleList so the state-dict keys are
    ``layers.{0,2,4,...}.{weight,bias}`` like the reference's."""

    def __init__(self, layers, nonlinearity, out_nonlinearity=None, normalize=False):
        super(DenseNet, self).__init__()
        if normalize:
            raise NotImplementedError('BatchNorm inside the edge MLP is used by no reference call site')
        self.n_layers = len(layers) - 1
        assert self.n_layers >= 1
        mods = []
        for j, (fan_in, fan_out) in enumerate(zip(layers[:-1], layers[1:])):
            mods.append(torch.nn.Linear(fan_in, fan_out))
            if j != self.n_layers - 1:
                mods.append(nonlinearity())
        if out_nonlinearity is not None:
            mods.append(out_nonlinearity())
        self.layers = torch.nn.ModuleList(mods)

    def forward(self, x):
        for layer in self.layers:
            x = layer(x)
        return x


class KernelNN(torch.nn.Module):
    def __init__(self, width, ker_width, depth, ker_in, in_width=1, out_width=1, relu_last=True, precision=None):
        super(KernelNN, self).__init__()
        self.depth = depth
        self.relu_last = relu_last
        self.fc1 = torch.nn.Linear(in_width, width)
        kernel = DenseNet([ker_in, ker_width, ker_width, width ** 2], torch.nn.ReLU)
        self.conv1 = NNConv_old(width, width, kernel, aggr='mean', precision=precision)
        self.fc2 = torch.nn.Linear(width, 1)

    def conv_stack(self, x, edge_index, edge_attr):
        """T applications of the ONE shared conv (UAI1_full_resolution.py:29-30); the edge features are
        computed on the first application and reused by the other T-1."""
        for k in range(self.depth):
            x = self.conv1(x, edge_index, edge_attr)
            if self.relu_last or k != self.depth - 1:
                x = F.relu(x)
        return x

    def forward(self, data):
        x, edge_index, edge_attr = data.x, data.edge_index, data.edge_attr
        x = self.fc1(x)
        x = self.conv_stack(x, edge_index, edge_attr)
        return self.fc2(x)


def _level_convs(width, ker_width, ker_in, levels, hidden, root_weight, bias, precision):
    convs = []
    for l in levels:
        kw = ker_width // (2 ** l)
        kernel = DenseNet([ker_in] + [kw] * hidden + [width ** 2], torch.nn.ReLU)
        convs.append(NNConv(width, width, kernel, aggr='mean', root_weight=root_weight, bias=bias,
                            precision=precision))
    return torch.nn.ModuleList(convs)


class _VCycleBase(torch.nn.Module):
    def _ranges(self, data):
        # one device->host copy for ALL slice bounds (the reference indexes with 0-d CUDA tensors: one
        # implicit sync per bound, ~40 per depth iteration -- SURVEY 3.3)
        # The cache entry HOLDS the three range tensors (so their storage cannot be freed and recycled for the
        # next sample's ranges) and is valid only for the same tensor objects at the same version.
        ts = (data.edge_index_down_range, data.edge_index_range, data.edge_index_up_range)
        hit = getattr(self, '_range_cache', None)
        if hit is None or any(a is not b for a, b in zip(hit[0], ts)) or hit[1] != tuple(t._version for t in ts):
            vals = tuple(t.tolist() for t in ts)
            hit = (ts, tuple(t._version for t in ts), vals)
            self._range_cache = hit
        return hit[2]


class KernelInduced(_VCycleBase):
    def __init__(self, width, ker_width, depth, ker_in, points, level, in_width=1, out_width=1, precision=None):
        super(KernelInduced, self).__init__()
        self.depth, self.width, self.level = depth, width, level
        self.points = points
        self.points_total = np.sum(points)
        self.fc_in = torch.nn.Linear(in_width, width)
        mk = lambda lv, hid: _level_convs(width, ker_width, ker_in, lv, hid, False, False, precision)  # noqa: E731
        self.conv_down_list = mk(range(1, level), 1)     # K12 K23 K34 (neurips1_MGKN.py:37-42)
        self.conv_list = mk(range(level), 2)             # K11 K22 K33 (:45-50)
        self.conv_up_list = mk(range(1, level), 1)       # K21 K32 K43 (:53-58)
        self.fc_out1 = torch.nn.Linear(width, ker_width)
        self.fc_out2 = torch.nn.Linear(ker_width, 1)

    def forward(self, data):
        r_down, r_mid, r_up = self._ranges(data)
        ei_d, ea_d = data.edge_index_down, data.edge_attr_down
        ei_m, ea_m = data.edge_index_mid, data.edge_attr_mid
        ei_u, ea_u = data.edge_index_up, data.edge_attr_up
        x = self.fc_in(data.x)
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()) or
                                                   any(t.requires_grad for t in (ea_d, ea_m, ea_u)))
        if _FUSED_STEPS and not needs_grad:
            # inference: the 13 * depth dependent steps  x <- relu(x + conv(x))  chained on pre-activations, ReLU and
            # residual inside each application's node-prep launch (NNConv_old.residual_step) -- 2 launches per step
            # instead of 5-6 in a chain that is launch-latency bound (SURVEY 8(f2))
            z, act = x, False
            for _ in range(self.depth):
                for l in range(self.level - 1):
                    a, b = r_down[l]
                    z, act = self.conv_down_list[l].residual_step(z, ei_d[:, a:b], ea_d[a:b, :], relu_in=act), True
                for l in reversed(range(self.level)):
                    a, b = r_mid[l]
                    z, act = self.conv_list[l].residual_step(z, ei_m[:, a:b], ea_m[a:b, :], relu_in=act), True
                    if l > 0:
                        a, b = r_up[l - 1]
                        z, act = self.conv_up_list[l - 1].residual_step(z, ei_u[:, a:b], ea_u[a:b, :], relu_in=act), True
            x = F.relu(z) if act else z
        else:
            for _ in range(self.depth):
                for l in range(self.level - 1):                                   # downward (:74-76)
                    a, b = r_down[l]
                    x = F.relu(x + self.conv_down_list[l](x, ei_d[:, a:b], ea_d[a:b, :]))
                for l in reversed(range(self.level)):                             # upward (:79-84)
                    a, b = r_mid[l]
                    x = F.relu(x + self.conv_list[l](x, ei_m[:, a:b], ea_m[a:b, :]))
                    if l > 0:
                        a, b = r_up[l - 1]
                        x = F.relu(x + self.conv_up_list[l - 1](x, ei_u[:, a:b], ea_u[a:b, :]))
        x = F.relu(self.fc_out1(x[:self.points[0]]))
        return self.fc_out2(x)


class MKGN(_VCycleBase):
    def __init__(self, width, ker_width, depth, ker_in, points, level, in_width=1, out_width=1, precision=None):
        super(MKGN, self).__init__()
        self.depth, self.width, self.level = depth, width, level
        self.points = [0] + [int(v) for v in np.cumsum(points)]              # MGKN_general_darcy2d.py:28-32
        self.points_total = np.sum(points)
        self.fc_in = torch.nn.Linear(in_width, width)
        self.conv_down_list = _level_convs(width, ker_width, ker_in, range(1, level), 1, False, False, precision)
        self.conv_list = _level_convs(width, ker_width, ker_in, range(level), 2, True, False, precision)   # :53
        self.conv_up_list = _level_convs(width, ker_width, ker_in, range(1, level), 1, False, False, precision)
        self.fc_out1 = torch.nn.Linear(width, ker_width)
        self.fc_out2 = torch.nn.Linear(ker_width, 1)
        self._rebased = {}

    def _mid_edges(self, data, l, a, b):
        """edge_index_mid[:, a:b] - points[l] (:85) computed once per graph instead of once per call."""
        ei = data.edge_index_mid
        hit = self._rebased.get(l)
        # the entry holds `ei` itself: same object + same version + same slice, or it is rebuilt
        if hit is None or hit[0] is not ei or hit[1] != (ei._version, a, b):
            hit = (ei, (ei._version, a, b), (ei[:, a:b] - self.points[l]).contiguous())
            self._rebased[l] = hit
        return hit[2]

    def forward(self, data):
        r_down, r_mid, r_up = self._ranges(data)
        ei_d, ea_d = data.edge_index_down, data.edge_attr_down
        ea_m = data.edge_attr_mid
        ei_u, ea_u = data.edge_index_up, data.edge_attr_up
        x = self.fc_in(data.x)
        for _ in range(self.depth):
            for l in range(self.level - 1):                                   # :77-80
                a, b = r_down[l]
                x = F.relu(x + self.conv_down_list[l](x, ei_d[:, a:b], ea_d[a:b, :]))
            for l in reversed(range(self.level)):                             # :83-90
                a, b = r_mid[l]
                lo, hi = self.points[l], self.points[l + 1]
                x = x.clone()
                x[lo:hi] = self.conv_list[l](x[lo:hi].clone(), self._mid_edges(data, l, a, b), ea_m[a:b, :])
                if l > 0:
                    a, b = r_up[l - 1]
                    x = F.relu(x + self.conv_up_list[l - 1](x, ei_u[:, a:b], ea_u[a:b, :]))
        x = F.relu(self.fc_out1(x[:self.points[1]]))
        return self.fc_out2(x)


class MGKN(torch.nn.Module):
    def __init__(self, width, ker_width, depth, ker_in, in_width, s, precision=None):
        super(MGKN, self).__init__()
        self.depth, self.width, self.s = depth, width, s
        self.level = int(np.log2(s) - 1)
        self.fc1 = torch.nn.Linear(in_width, width)
        convs = []
        for l in range(self.level + 1):                                       # MGKN_orthogonal_burgers1d.py:33-38
            kw = max(ker_width // (2 ** l), 16)
            kernel = DenseNet([ker_in, kw, kw, width ** 2], torch.nn.ReLU)
            convs.append(NNConv(width, width, kernel, aggr='mean', precision=precision))
        self.conv_list = torch.nn.ModuleList(convs)
        self.fc2 = torch.nn.Linear(width, ker_width)
        self.fc3 = torch.nn.Linear(ker_width, 1)

    def Upsample(self, x, channels, scale, s):                                # :45-49
        x = x.transpose(0, 1).reshape(1, channels, s)
        x = F.interpolate(x, scale_factor=scale, mode='nearest')
        return x.reshape(channels, -1).transpose(0, 1)

    def Downsample(self, x, channels, scale, s):                              # :52-56
        x = x.transpose(0, 1).reshape(1, channels, s)
        x = F.avg_pool1d(x, kernel_size=scale)
        return x.reshape(channels, -1).transpose(0, 1)

    def forward(self, data):
        X_list, _, edge_index_list, edge_attr_list = data
        level = len(X_list)
        x = self.fc1(X_list[0])
        phi = [None] * level
        for _ in range(self.depth):
            for l in range(level):                                            # restriction (:67-71)
                phi[l] = x
                if l != level - 1:
                    x = self.Downsample(x, self.width, 2, self.s // (2 ** l))
            x = F.relu(x + self.conv_list[-1](phi[-1], edge_index_list[-1], edge_attr_list[-1]))   # :74
            for l in reversed(range(level)):
                if l != 0:
                    x = self.Upsample(x, self.width, 2, self.s // (2 ** l))                          # :78
                    x = F.relu(x + self.conv_list[l](phi[l - 1], edge_index_list[l], edge_attr_list[l]))
                else:
                    x = F.relu(x + self.conv_list[0](phi[0], edge_index_list[0], edge_attr_list[0]))
        x = F.relu(self.fc2(x))
        return self.fc3(x)
