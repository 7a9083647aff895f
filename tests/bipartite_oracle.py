"""fp64 restatement of the bipartite NNConv (DESIGN 4.10), differentiable with autograd:

    out[i] = x_dst[i] root + bias + aggr_{e: dst_e = i} x_src[src_e] . nn(e).view(in_src, out)

over N_dst target rows; edge_index row 0 indexes x_src, row 1 x_dst.  aggr 'add', 'mean' (in-degree over the targets,
1/max(deg, 1)) or 'max' (per channel; a target without in-edges gets 0).  x_dst None drops the root term.  The edge
network is Linear (act Linear)*, given as fp64 weight / bias lists."""
import torch


def edge_network(ea, ws, bs, act=torch.relu):
    h = ea.double()
    for w, b in zip(ws[:-1], bs[:-1]):
        h = act(h @ w.double().t() + b.double())
    return h @ ws[-1].double().t() + bs[-1].double()


def bipartite_forward(x_src, x_dst, edge_index, edge_attr, ws, bs, root, bias, aggr, n_dst, act=torch.relu):
    src, dst = edge_index[0].long(), edge_index[1].long()
    x_src = x_src.double()
    in_src = x_src.size(1)
    k = edge_network(edge_attr, ws, bs, act)
    cout = k.size(1) // in_src
    msg = torch.einsum('ei,eio->eo', x_src[src], k.view(-1, in_src, cout))
    out = torch.zeros(n_dst, cout, dtype=torch.float64, device=msg.device)
    if aggr == 'max':
        idx = dst.unsqueeze(1).expand(-1, cout)
        out = out.scatter_reduce(0, idx, msg, reduce='amax', include_self=False)
    else:
        out = out.index_add(0, dst, msg)
        if aggr == 'mean':
            deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).double()
            out = out / deg.unsqueeze(1)
    if x_dst is not None and root is not None:
        out = out + x_dst.double() @ root.double()
    if bias is not None:
        out = out + bias.double()
    return out
