"""Multi-GPU decomposition of the NNConv path (SURVEY 8(e)); the reference itself is single-GPU.

Two ways the path shards, both one process per GPU over torch.distributed (NCCL on GPUs, gloo in
the CPU tests):

1. **Batch sharding** (BASELINE config 3): graphs of a training / inference batch are independent connected
   components, so rank r owns graphs g with g % world == r.  Forward has NO data-path collective; training
   adds one all-reduce of parameter gradients per step.  ``shard_indices`` + ``allreduce_gradients``.

2. **Node-range cuts of one big mesh** (config 3 alt. / 5): the square grid is row-major (node = iy*s + ix,
   graph-neural-operator/utilities.py:248), so contiguous node ranges are horizontal strips.  A ball of
   radius r reaches R = floor(r*(s-1)) grid rows, hence a rank needs R halo rows above and below its strip;
   edges are assigned to the owner of their DESTINATION so the scatter stays local, and ONE halo exchange
   (all-gather of every rank's 2R boundary rows) precedes each of the T conv applications.
   ``StripPartition`` builds the local sub-graph with the reference's edge order, ``halo_exchange`` moves the
   boundary rows.
"""
import ctypes
import math

import torch
import torch.distributed as dist

from . import graphs


def shard_indices(n_items, rank, world):
    """Round-robin ownership of independent graphs: item g belongs to rank g % world."""
    return list(range(rank, n_items, world))


def allreduce_gradients(module, group=None):
    """Sum-reduce parameter gradients across ranks (the reference's losses are sums over the batch,
    UAI1_full_resolution.py:265, so no rescale).  One flat all-reduce: ~21 MB for KernelNN(w=64, kw=1024)."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    # EVERY rank reduces the same flat buffer: all trainable parameters in module order, zeros standing in for a
    # missing .grad (a rank with an empty shard or an unused parameter must not shorten the buffer)
    params = [p for p in module.parameters() if p.requires_grad]
    if not params:
        return
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1).float() for p in params])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    off = 0
    for p in params:
        n = p.numel()
        g = flat[off:off + n].view_as(p).to(p.dtype)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n


class StripPartition(object):
    """Horizontal-strip partition of the s x s ball graph for one rank.

    Local node numbering: [halo_above | owned | halo_below] (global order preserved), so local index =
    global index - first_local_global.  ``edge_index`` (local numbering, int64 [2, E_loc]) holds every edge
    whose destination is owned, in the reference's source-major order; ``edge_ids`` are not needed because
    edge attributes are recomputed from positions / theta exactly like the reference does per sample.
    """

    def __init__(self, s, r, rank, world, device='cpu', ties_in=True):
        self.s, self.r, self.rank, self.world = s, r, rank, world
        self.R = int(math.floor(r * (s - 1) + 1e-9))
        rows = [(s * k) // world for k in range(world + 1)]          # row ranges per rank
        self.row_lo, self.row_hi = rows[rank], rows[rank + 1]
        self.all_rows = rows
        if min(b - a for a, b in zip(rows[:-1], rows[1:])) < self.R:
            raise ValueError('strips thinner than the ball radius need multi-hop halos (not built)')
        self.halo_lo = max(0, self.row_lo - self.R)
        self.halo_hi = min(s, self.row_hi + self.R)
        self.first = self.halo_lo * s                                  # global id of local node 0
        self.n_local = (self.halo_hi - self.halo_lo) * s
        self.own_lo = (self.row_lo - self.halo_lo) * s                # local range of owned nodes
        self.own_hi = self.own_lo + (self.row_hi - self.row_lo) * s
        ei = graphs.ball_connectivity(s, r, device, ties_in, nodes=(self.halo_lo * s, self.halo_hi * s))
        keep = (ei[1] >= self.row_lo * s) & (ei[1] < self.row_hi * s)  # destination owned
        self.edge_index_global = ei[:, keep]
        self.edge_index = self.edge_index_global - self.first

    def local_slice(self, x_global):
        return x_global[self.first:self.first + self.n_local]

    def boundary_rows(self, x_local):
        """The 2R owned grid rows (top R, bottom R) other ranks may need: [2R*s, C]."""
        s, R = self.s, self.R
        top = x_local[self.own_lo:self.own_lo + R * s]
        bot = x_local[self.own_hi - R * s:self.own_hi]
        return torch.cat([top, bot], dim=0)


def halo_exchange(x_local, part, group=None):
    """Refresh the halo rows of x_local in place from the neighbours' boundary rows.
    One all-gather of [2R*s, C] per rank (740 KB per side at 241^2, r=0.05, C=64 fp32)."""
    s, R = part.s, part.R
    send = part.boundary_rows(x_local).contiguous()
    if part.world == 1:
        return x_local
    bufs = [torch.empty_like(send) for _ in range(part.world)]
    dist.all_gather(bufs, send, group=group)
    # halo above = bottom R rows of rank-1 ; halo below = top R rows of rank+1
    n_above = (part.row_lo - part.halo_lo) * s
    if n_above > 0:
        x_local[:n_above] = bufs[part.rank - 1][R * s:][-n_above:]
    n_below = (part.halo_hi - part.row_hi) * s
    if n_below > 0:
        x_local[part.own_hi:part.own_hi + n_below] = bufs[part.rank + 1][:R * s][:n_below]
    return x_local


def partitioned_conv_stack(conv_fn, x_local, part, edge_attr_local, depth, relu_last=True, group=None):
    """T applications of a shared conv on one rank's strip.  ``conv_fn(x, edge_index, edge_attr) -> [n_local,
    C]`` computes rows for every local node but only OWNED rows are meaningful (edges end in owned nodes);
    halo rows are overwritten by the exchange before the next application."""
    x = x_local
    for k in range(depth):
        out = conv_fn(x, part.edge_index, edge_attr_local)
        if relu_last or k != depth - 1:
            out = torch.relu(out)
        x = out
        if k != depth - 1:
            x = halo_exchange(x, part, group)
    return x[part.own_lo:part.own_hi]


# ------------------------------------------------------------------------------------------------------
# Halo exchange by peer stores over NVLink (csrc/halo.cu): no NCCL call and no host round trip between the T
# applications of the conv stack.
# ------------------------------------------------------------------------------------------------------
def halo_ranges(part):
    """Which of this rank's local rows go where: dict with, per direction, (src_row0, dst_row0, n_rows) in units of
    NODES -- src in this rank's local numbering, dst in the NEIGHBOUR's local numbering.  'up' = rank-1 (its halo
    below its strip receives my top R grid rows), 'down' = rank+1 (its halo above receives my bottom R grid rows)."""
    s, R = part.s, part.R
    rows = part.all_rows
    out = {'up': None, 'down': None}
    if part.rank > 0:
        up_lo, up_hi = rows[part.rank - 1], rows[part.rank]
        up_halo_lo = max(0, up_lo - R)
        up_own_hi = (up_hi - up_halo_lo) * s                       # neighbour's local index of its first halo-below node
        n = min(s, up_hi + R) - up_hi                              # grid rows the neighbour has below its strip
        out['up'] = (part.own_lo, up_own_hi, n * s)
    if part.rank < part.world - 1:
        dn_lo = rows[part.rank + 1]
        dn_halo_lo = max(0, dn_lo - R)
        n = dn_lo - dn_halo_lo                                     # grid rows the neighbour has above its strip
        out['down'] = (part.own_hi - n * s, 0, n * s)
    return out


class _DevMem(object):
    """Zero-copy torch view of raw device memory (``torch.as_tensor`` reads __cuda_array_interface__)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (int(ptr), False), 'version': 2}


class PeerHalo(object):
    """Double-buffered node-feature buffers of one rank plus one flag word per direction, in ONE peer-visible
    allocation (``nnconv_ipc_alloc``) that the two neighbours map with CUDA IPC (``nnconv_ipc_open``, opened with the
    importing rank's device current so that its kernels may store into it).  ``advance(out, k)`` turns the result of
    application k into the input of application k+1: ReLU + copy of the owned rows + peer stores of the boundary rows
    + flag (one small kernel pair), then a one-thread wait kernel for the neighbours' flags.  Everything is
    stream-ordered on the device; no NCCL call between the applications."""

    def __init__(self, part, channels, device, group=None):
        from . import _lib
        self.part, self.C, self.dev, self.group = part, channels, device, group
        self.L = _lib.lib()
        self._lib = _lib
        self.buf_bytes = ((part.n_local * channels * 4 + 255) // 256) * 256
        nbytes = 2 * self.buf_bytes + 256
        handle = ctypes.create_string_buffer(64)
        ptr = ctypes.c_void_p()
        with torch.cuda.device(device):
            _lib.check(self.L.nnconv_ipc_alloc(nbytes, ctypes.byref(ptr), handle))
        self.base = ptr.value
        raw = torch.as_tensor(_DevMem(self.base, nbytes), device=device)
        self.bufs = [raw[i * self.buf_bytes:i * self.buf_bytes + part.n_local * channels * 4].view(torch.float32)
                     .view(part.n_local, channels) for i in range(2)]
        self.flags_ptr = self.base + 2 * self.buf_bytes                       # int32 [from_up, from_down]
        gathered = [None] * part.world
        dist.all_gather_object(gathered, (bytes(handle.raw), self.buf_bytes), group=group)
        self._opened = []

        def open_(r):
            h, bb = gathered[r]
            p = ctypes.c_void_p()
            with torch.cuda.device(device):
                _lib.check(self.L.nnconv_ipc_open(h, ctypes.byref(p)))
            self._opened.append(p.value)
            return dict(bufs=[p.value, p.value + bb], flags=p.value + 2 * bb)
        self.up = open_(part.rank - 1) if part.rank > 0 else None
        self.down = open_(part.rank + 1) if part.rank < part.world - 1 else None
        self.ranges = halo_ranges(part)
        self.seq = 0
        dist.barrier(group=group)

    def close(self):
        """Unmap the neighbours' buffers and free this rank's (collective: everybody unmaps before anybody frees)."""
        if self.base is None:
            return
        torch.cuda.synchronize(self.dev)
        for p in self._opened:
            self.L.nnconv_ipc_close(ctypes.c_void_p(p))
        self._opened = []
        dist.barrier(group=self.group)
        self.bufs = None
        self.L.nnconv_ipc_free(ctypes.c_void_p(self.base))
        self.base = None

    def load(self, x_local):
        """Input of application 0 (halo rows already correct: every rank slices the same global tensor)."""
        self.bufs[0].copy_(x_local)
        return self.bufs[0]

    def _push(self, out_ptr, relu, own_lo, own_hi, nxt_ptr, k_next, up, dn):
        st = torch.cuda.current_stream(self.dev).cuda_stream
        vp = ctypes.c_void_p
        u = up or (0, 0, 0)
        d = dn or (0, 0, 0)
        # my rows land in the neighbour ABOVE as its "from_down" halo / flag, in the neighbour BELOW as its "from_up"
        self._lib.check(self.L.nnconv_halo_push(
            vp(out_ptr), 1 if relu else 0, self.part.n_local, self.C, own_lo, own_hi, vp(nxt_ptr),
            vp(self.up['bufs'][k_next]) if up else vp(0), u[0], u[1], u[2],
            vp(self.down['bufs'][k_next]) if dn else vp(0), d[0], d[1], d[2],
            vp(self.up['flags'] + 4) if up else vp(0), vp(self.down['flags']) if dn else vp(0), self.seq, vp(st)))
        self._lib.check(self.L.nnconv_halo_wait(vp(self.flags_ptr) if up else vp(0), vp(self.flags_ptr + 4) if dn else vp(0),
                                                self.seq, vp(st)))

    def advance(self, out, k, relu=True):
        nxt = self.bufs[(k + 1) % 2]
        self.seq += 1
        p = self.part
        self._push(out.data_ptr(), relu, p.own_lo, p.own_hi, nxt.data_ptr(), (k + 1) % 2, self.ranges['up'], self.ranges['down'])
        return nxt

    def finish(self):
        """End-of-stack handshake (flags only): returns once both neighbours have retired their last application,
        so the next stack's pushes cannot overwrite halo rows a slower neighbour is still reading."""
        self.seq += 1
        b = self.bufs[0].data_ptr()
        up = (0, 0, 0) if self.up else None
        dn = (0, 0, 0) if self.down else None
        self._push(b, False, 0, 0, b, 0, up, dn)


def partitioned_conv_stack_peer(conv_fn, x_local, part, edge_attr_local, depth, halo, relu_last=True):
    """Same as partitioned_conv_stack with the halo moved by peer stores (PeerHalo) instead of an all-gather."""
    x = halo.load(x_local)
    for k in range(depth):
        out = conv_fn(x, part.edge_index, edge_attr_local)
        relu = relu_last or k != depth - 1
        if k != depth - 1:
            x = halo.advance(out, k, relu)
        else:
            x = torch.relu(out) if relu else out
    halo.finish()
    return x[part.own_lo:part.own_hi]


# ------------------------------------------------------------------------------------------------------
# 1-D aligned node-range partition of the multipole hierarchy (BASELINE config 5: orthogonal MGKN, Burgers 1-D,
# multipole-graph-neural-operator/MGKN_orthogonal_burgers1d.py:59-86 on multi_pole_grid1d, utilities.py:1702-1769)
# ------------------------------------------------------------------------------------------------------
class Range1DPartition(object):
    """Rank r owns the finest-level nodes [lo, hi) with lo, hi multiples of 2^(levels-1), hence nodes
    [lo >> j, hi >> j) of level j: avg_pool1d(2) restriction and nearest-neighbour prolongation stay local.  The
    stencils reach |offset| <= 3 (utilities.py:1749), so every level carries ``halo`` = 3 nodes per side
    (periodic wrap when the mesh is periodic); edges are owned by their DESTINATION.  Local layout per level:
    [halo_left | owned | halo_right]."""

    def __init__(self, s, levels, rank, world, halo=3, periodic=True):
        self.s, self.levels, self.rank, self.world, self.halo, self.periodic = s, levels, rank, world, halo, periodic
        align = 2 ** (levels - 1)
        blocks = s // align
        cuts = [(blocks * k) // world * align for k in range(world + 1)]
        self.lo, self.hi = cuts[rank], cuts[rank + 1]
        if min(b - a for a, b in zip(cuts[:-1], cuts[1:])) >> (levels - 1) < halo:
            raise ValueError('ranges narrower than the halo on the coarsest level')

    def owned(self, j):
        return self.lo >> j, self.hi >> j

    def n_local(self, j):
        a, b = self.owned(j)
        return (b - a) + 2 * self.halo

    def local_edges(self, j, edge_index):
        """Edges of level j that END in an owned node, in the global order, renumbered locally.  Returns
        (edge_index_local, mask) -- mask selects the matching rows of edge_attr."""
        a, b = self.owned(j)
        n = self.s >> j
        mask = (edge_index[1] >= a) & (edge_index[1] < b)
        e = edge_index[:, mask]
        base = a - self.halo
        loc = (e - base) % n if self.periodic else (e - base)
        return loc.contiguous(), mask

    def with_halos(self, owned_rows, group=None):
        """owned_rows: list over levels of [owned_j, C] tensors -> list of [halo + owned_j + halo, C]; ONE
        all-gather of every level's 2*halo boundary rows."""
        h = self.halo
        send = torch.cat([torch.cat([x[:h], x[-h:]], dim=0) for x in owned_rows], dim=0).contiguous()
        if self.world > 1:
            bufs = [torch.empty_like(send) for _ in range(self.world)]
            dist.all_gather(bufs, send, group=group)
        else:
            bufs = [send]
        left, right = bufs[(self.rank - 1) % self.world], bufs[(self.rank + 1) % self.world]
        out = []
        for j, x in enumerate(owned_rows):
            o = 2 * h * j
            hl = left[o + h:o + 2 * h]          # the left neighbour's LAST h owned rows
            hr = right[o:o + h]                 # the right neighbour's FIRST h owned rows
            if not self.periodic:
                if self.rank == 0:
                    hl = torch.zeros_like(hl)
                if self.rank == self.world - 1:
                    hr = torch.zeros_like(hr)
            out.append(torch.cat([hl, x, hr], dim=0))
        return out


def partitioned_mgkn_forward(part, X0_owned, edge_index_local, edge_attr_local, convs, fc1, fc2, fc3, depth, width,
                             group=None):
    """MGKN.forward (MGKN_orthogonal_burgers1d.py:59-86) on one rank's node range.  ``convs[l](x_local, ei, ea)``
    returns [n_local, width] (owned rows valid); ``edge_index_local[l]`` / ``edge_attr_local[l]`` come from
    ``part.local_edges``: set l >= 1 acts on level l-1, set 0 on level 0, the LAST set on the coarsest level.
    One halo exchange (all levels in one all-gather) per depth iteration; restriction / prolongation are local."""
    import torch.nn.functional as F
    level = len(edge_index_local) - 1
    h = part.halo

    def down(x):
        return F.avg_pool1d(x.t().unsqueeze(0), kernel_size=2).squeeze(0).t()

    def up(x):
        return x.repeat_interleave(2, dim=0)

    def own(t):
        return t[h:t.size(0) - h]
    x = fc1(X0_owned)
    for _ in range(depth):
        phi = []
        for l in range(level):
            phi.append(x)
            if l != level - 1:
                x = down(x)
        phi_h = part.with_halos(phi, group)                        # the only communication of the iteration
        x = torch.relu(x + own(convs[-1](phi_h[-1], edge_index_local[-1], edge_attr_local[-1])))
        for l in reversed(range(level)):
            if l != 0:
                x = up(x)
                x = torch.relu(x + own(convs[l](phi_h[l - 1], edge_index_local[l], edge_attr_local[l])))
            else:
                x = torch.relu(x + own(convs[0](phi_h[0], edge_index_local[0], edge_attr_local[0])))
    return fc3(torch.relu(fc2(x)))
