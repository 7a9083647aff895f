"""Input side of the NNConv path: radius ("ball") graphs of a regular square mesh, built without the
reference's dense O(N^2) distance matrix.

Reference being mirrored: ``SquareMeshGenerator`` (graph-neural-operator/utilities.py:229-285):
``ball_connectivity(r)`` = ``np.vstack(np.where(pairwise_distances(grid) <= r))`` (:250-255) and
``attributes(theta=...)`` = ``[pos_src, pos_dst, theta_src, theta_dst]`` (:269-277).  The reference cannot
build the 241 x 241 graph (27 GB distance matrix); here edges are enumerated per node from the integer
lattice stencil, on whatever device is asked (torch ops only -- this is input generation, not the hot path).

Edge ORDER is the reference's: source-major, destination ascending (np.where row-major order).
TIE RULE (SURVEY H3): lattice offsets whose distance equals r exactly (e.g. (+-12, 0) at s=241, r=0.05)
are decided in exact integer arithmetic: included when ``ties_in`` (mathematical <=), excluded otherwise;
sklearn's float64 expanded-form distance decides them by rounding noise.
"""
import math

import torch


def ball_offsets(s, r, ties_in=True):
    rr = r * (s - 1)
    lim2 = rr * rr
    big = int(math.floor(rr + 1e-9))
    offs = []
    for dy in range(-big, big + 1):
        for dx in range(-big, big + 1):
            d2 = dx * dx + dy * dy
            on_sphere = abs(d2 - lim2) <= 1e-9 * max(lim2, 1.0)
            if (d2 < lim2 and not on_sphere) or (on_sphere and ties_in):
                offs.append((dy, dx))
    return offs      # sorted by (dy, dx): ascending destination index for a fixed source


def square_grid(s, device='cpu', dtype=torch.float32):
    """utilities.py:241-248: node = iy*s + ix, position (ix/(s-1), iy/(s-1)) (np.meshgrid 'xy' order)."""
    lin = torch.linspace(0.0, 1.0, s, dtype=torch.float64, device=device)
    gy, gx = torch.meshgrid(lin, lin, indexing='ij')
    return torch.stack([gx.reshape(-1), gy.reshape(-1)], dim=1).to(dtype)


def ball_connectivity(s, r, device='cpu', ties_in=True, node_chunk=1 << 16, nodes=None):
    """edge_index [2, E] int64 on `device`, source-major / destination-ascending.
    nodes=(n0, n1) restricts the SOURCE nodes to [n0, n1) (used to cut bounded samples of a big graph)."""
    offs = torch.tensor(ball_offsets(s, r, ties_in), dtype=torch.int64, device=device)   # [K, 2] (dy, dx)
    n_lo, n = (0, s * s) if nodes is None else (int(nodes[0]), min(int(nodes[1]), s * s))
    out = []
    for n0 in range(n_lo, n, node_chunk):
        node = torch.arange(n0, min(n, n0 + node_chunk), dtype=torch.int64, device=device)
        iy, ix = node // s, node % s
        jy = iy[:, None] + offs[None, :, 0]
        jx = ix[:, None] + offs[None, :, 1]
        ok = (jy >= 0) & (jy < s) & (jx >= 0) & (jx < s)
        src = node[:, None].expand_as(jy)[ok]
        dst = (jy * s + jx)[ok]
        out.append(torch.stack([src, dst]))
    return torch.cat(out, dim=1)


def ball_edge_attr(grid, edge_index, theta):
    """utilities.py:269-277: edge_attr[e] = (pos_src(2), pos_dst(2), theta_src, theta_dst), fp32."""
    src, dst = edge_index[0], edge_index[1]
    theta = theta.to(grid.dtype)
    return torch.cat([grid[src], grid[dst], theta[src, None], theta[dst, None]], dim=1).float().contiguous()


def darcy_sample(s, r, device='cpu', seed=0, edge_index=None, ties_in=True):
    """Synthetic Darcy-2D sample with the shapes of UAI1_full_resolution.py:143-159: node features
    x [N,6] = (grid xy, a, a_smooth, a_gradx, a_grady) ~ N(0,1) stand-ins, edge_attr [E,6]."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    grid = square_grid(s, device)
    feats = torch.randn(s * s, 4, generator=g).to(device)
    if edge_index is None:
        edge_index = ball_connectivity(s, r, device, ties_in)
    x = torch.cat([grid, feats], dim=1).contiguous()
    edge_attr = ball_edge_attr(grid, edge_index, feats[:, 0])
    return x, edge_index, edge_attr


# ------------------------------------------------------------------------------------------------------
# Multi-level (MGKN) graphs: RandomMultiMeshGenerator restated (multipole-graph-neural-operator/
# utilities.py:546-712) with torch ops on any device.
# ------------------------------------------------------------------------------------------------------
def ball_pairs_device(pa, pb, radius, src_base=0, dst_base=0, theta_a=None, theta_b=None, with_attr=False):
    """np.vstack(np.where(pairwise_distances(pa, pb) <= radius)) on the GPU without the N x N matrix: the
    hand-written count / fill kernels of csrc/graph_build.cu (one thread per source point walks the destination
    points in ascending order, so the row-major edge order needs no sort).  pa [na,2], pb [nb,2] CUDA tensors.
    Returns edge_index [2,E] int64 (ids offset by src_base / dst_base) and, with_attr, edge_attr [E, 4 | 6] fp32 =
    [pos_src, pos_dst (, theta_src, theta_dst)] (utilities.py:269-285 / multipole utilities.py:672-706)."""
    import ctypes

    from . import _lib
    L = _lib.lib()
    dev = pa.device
    pa64 = pa.detach().to(torch.float64).contiguous()
    pb64 = pb.detach().to(torch.float64).contiguous()
    na, nb = pa64.size(0), pb64.size(0)
    vp = ctypes.c_void_p
    with torch.cuda.device(dev):
        st = vp(torch.cuda.current_stream(dev).cuda_stream)
        counts = torch.empty(max(na, 1), dtype=torch.int32, device=dev)
        _lib.check(L.nnconv_ball_count(vp(pa64.data_ptr()), na, vp(pb64.data_ptr()), nb, float(radius),
                                       vp(counts.data_ptr()), st))
        incl = torch.cumsum(counts[:na].to(torch.int64), 0)
        e = int(incl[-1].item()) if na > 0 else 0            # one host read per graph (the edge count sizes the output)
        offsets = (incl - counts[:na]).contiguous()
        ei = torch.empty(2, e, dtype=torch.int64, device=dev)
        ta = theta_a.detach().to(torch.float64).contiguous() if theta_a is not None else None
        tb = theta_b.detach().to(torch.float64).contiguous() if theta_b is not None else None
        attr = torch.empty(e, 6 if ta is not None else 4, dtype=torch.float32, device=dev) if with_attr else None
        if e > 0:
            _lib.check(L.nnconv_ball_fill(vp(pa64.data_ptr()), na, vp(pb64.data_ptr()), nb, float(radius),
                                          vp(offsets.data_ptr()), int(src_base), int(dst_base), vp(ei[0].data_ptr()),
                                          vp(ei[1].data_ptr()), vp(ta.data_ptr()) if ta is not None else vp(0),
                                          vp(tb.data_ptr()) if tb is not None else vp(0),
                                          vp(attr.data_ptr()) if attr is not None else vp(0), st))
    return (ei, attr) if with_attr else ei


def _ball_pairs(pa, pb, radius):
    """np.vstack(np.where(pairwise_distances(pa, pb) <= radius)): row-major order = source-major, dst ascending.
    Float64 distances; lattice ties with `radius` are rounding-dependent in the reference too (SURVEY H3).
    CUDA tensors go through the device kernels (no N x N matrix); the dense torch.cdist form is the CPU path used
    by the host-side tests."""
    if pa.is_cuda:
        return ball_pairs_device(pa, pb, radius)
    d = torch.cdist(pa.double(), pb.double())
    idx = torch.nonzero(d <= radius, as_tuple=False)
    return idx.t().contiguous()


class MultiLevelGraph(object):
    """Output of ``multi_level_ball_graph`` with the field names the MGKN scripts put on their ``Data``
    (neurips1_MGKN.py:208-224): edge_index_{mid,down,up} (concatenated over levels, global node ids),
    edge_index_range / _down_range / _up_range ([L,2] / [L-1,2]), edge_attr_{mid,down,up}, sample_idx."""
    pass


def multi_level_ball_graph(s, sample_sizes, radius_inner, radius_inter, theta=None, device='cpu', generator=None):
    """sample(): one torch.randperm(s*s) split into consecutive level chunks (utilities.py:581-593);
    ball_connectivity(): per-level ball graphs offset by the level's first node id, inter-level bipartite graphs
    level l -> l+1 ("down") and their transposes ("up") (:602-643); attributes(): [pos_src, pos_dst,
    theta_src, theta_dst] (:672-706).  theta: [s*s] tensor or None (then edge_attr has 4 columns)."""
    level = len(sample_sizes)
    assert len(radius_inner) == level and len(radius_inter) == level - 1
    grid = square_grid(s, 'cpu', torch.float64)
    perm = torch.randperm(s * s, generator=generator)
    idx, pos, start = [], [], [0]
    off = 0
    for m in sample_sizes:
        idx.append(perm[off:off + m])
        pos.append(grid[idx[-1]].to(device))
        off += m
        start.append(off)
    idx_all = perm[:off]
    pos_all = grid[idx_all].to(device)
    mid, down, up = [], [], []
    for l in range(level):
        mid.append(_ball_pairs(pos[l], pos[l], radius_inner[l]) + start[l])
    for l in range(level - 1):
        e = _ball_pairs(pos[l], pos[l + 1], radius_inter[l])
        e = torch.stack([e[0] + start[l], e[1] + start[l + 1]])
        down.append(e)
        up.append(e[[1, 0], :])

    def ranges(parts):
        r, n = [], 0
        for p in parts:
            r.append([n, n + p.size(1)])
            n += p.size(1)
        return torch.tensor(r, dtype=torch.long)

    def attrs(e):
        cols = [pos_all[e[0]], pos_all[e[1]]]
        if theta is not None:
            th = theta.to(device).double()[idx_all.to(device)]
            cols += [th[e[0], None], th[e[1], None]]
        return torch.cat(cols, dim=1).float().contiguous()

    g = MultiLevelGraph()
    g.sample_idx = idx_all
    g.points = list(sample_sizes)
    g.pos = pos_all.float()
    g.edge_index_mid = torch.cat(mid, dim=1)
    g.edge_index_down = torch.cat(down, dim=1)
    g.edge_index_up = torch.cat(up, dim=1)
    g.edge_index_range, g.edge_index_down_range, g.edge_index_up_range = ranges(mid), ranges(down), ranges(up)
    g.edge_attr_mid, g.edge_attr_down, g.edge_attr_up = attrs(g.edge_index_mid), attrs(g.edge_index_down), attrs(g.edge_index_up)
    return g


# ------------------------------------------------------------------------------------------------------
# 1-D multipole hierarchy (orthogonal MGKN, Burgers): multi_pole_grid1d restated
# (multipole-graph-neural-operator/utilities.py:1702-1768), vectorised, any device.
# ------------------------------------------------------------------------------------------------------
def multi_pole_grid1d(theta, s, is_periodic=False, levels=None, device='cpu'):
    """theta: [s] coefficient of ONE sample on the finest grid.  Returns (X_list, edge_index_list, edge_attr_list):
    level l (1-based) has s_l = s / 2^(l-1) nodes at linspace(0,1,s_l) with theta subsampled by stride 2^(l-1);
    edge set 0 = nearest neighbours of the finest level (offsets -1,+1), edge set l = 'interactive' neighbours of
    level l (offsets -3..3 with |offset| >= 2 whose parents are adjacent: |x_i//2 - x_j//2| mod (s_l/2) <= 1), in
    the reference's (x_i major, offset ascending) order.  edge_attr = [x_src, x_dst, theta_src, theta_dst]
    (get_edge_attr, utilities.py:1771-1777); X_l = [x, theta_l].  `levels` truncates the hierarchy (the shipped
    rule int(log2 s - 1) gives 12 levels at s=8192; BASELINE config 5 names 5)."""
    n_levels = int(math.log2(s) - 1)
    if levels is not None:
        n_levels = min(n_levels, int(levels))
    theta = torch.as_tensor(theta).reshape(-1).to(device)

    def pairs(s_l, offsets, inter):
        xi = torch.arange(s_l, device=device)[:, None].expand(s_l, len(offsets))
        off = torch.tensor(offsets, device=device)[None, :].expand(s_l, len(offsets))
        xj = xi + off
        if is_periodic:
            xj = xj % s_l
            ok = torch.ones_like(xj, dtype=torch.bool)
        else:
            ok = (xj >= 0) & (xj < s_l)
        if inter:
            par = (torch.div(xi, 2, rounding_mode='floor') - torch.div(xj, 2, rounding_mode='floor')).abs()
            ok = ok & (par % (s_l // 2) <= 1)
        return torch.stack([xi[ok], xj[ok]]).long()

    X_list, ei_list, ea_list = [], [], []
    for l in range(1, n_levels + 1):
        r_l = 2 ** (l - 1)
        s_l = s // r_l
        grid_l = torch.linspace(0.0, 1.0, s_l, dtype=torch.float64, device=device).float()
        theta_l = theta[::r_l][:s_l].float()
        X_list.append(torch.stack([grid_l, theta_l], dim=1))

        def attr(e):
            return torch.stack([grid_l[e[0]], grid_l[e[1]], theta_l[e[0]], theta_l[e[1]]], dim=1).contiguous()

        if l == 1:
            e = pairs(s_l, [-1, 1], False)
            ei_list.append(e)
            ea_list.append(attr(e))
        e = pairs(s_l, [-3, -2, 2, 3], True)
        ei_list.append(e)
        ea_list.append(attr(e))
    return X_list, ei_list, ea_list


def grid_edge(n_x, n_y, device='cpu'):
    """The lattice of MGNO/utilities.py:1480-1520 (``grid_edge(n_x, n_y)``, a = None), vectorised: returns
    (grid [n_x n_y, 2] fp32, edge_index [2, E] int64).  Node i = y n_x + x sits at (x / (n_x - 1), y / (n_y - 1)); node
    by node in that order, the edges are (i, i+1), (i+1, i) unless x is the last column, then (i, i+n_x), (i+n_x, i)
    unless y is the last row -- the reference's edge order."""
    xs = torch.linspace(0.0, 1.0, n_x, dtype=torch.float64)
    ys = torch.linspace(0.0, 1.0, n_y, dtype=torch.float64)
    gy, gx = torch.meshgrid(ys, xs, indexing='ij')
    grid = torch.stack([gx.reshape(-1), gy.reshape(-1)], dim=1).float().to(device)
    i = torch.arange(n_x * n_y, dtype=torch.int64, device=device)
    x, y = i % n_x, i // n_x
    pairs = torch.stack([torch.stack([i, i + 1], 1), torch.stack([i + 1, i], 1),
                         torch.stack([i, i + n_x], 1), torch.stack([i + n_x, i], 1)], dim=1)   # [N, 4, 2]
    ok = torch.stack([x != n_x - 1, x != n_x - 1, y != n_y - 1, y != n_y - 1], dim=1)       # [N, 4]
    return grid, pairs[ok].t().contiguous()
