"""Drop-in for the reference's ``models/tensor_layers.py``: same class name, constructor keywords, ``forward``
signature and ``state_dict`` keys (``fc.{g}.{0,3}.weight/bias``, ``batch_norm.{weight,bias,running_mean,running_var}``),
with the convolution executed by the fused sm_90a kernel (csrc/tpconv.cu) instead of
e3nn + torch_scatter (models/tensor_layers.py:125-231,309-335).

Inference only (eval-mode BatchNorm, dropout = identity); CUDA only - there is no CPU fallback.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import fused, ops, radial
from .irreps import irreps_dim, parse_irreps
from .tp_table import build_table

ACTIVATIONS = {'relu': nn.ReLU, 'silu': nn.SiLU}

# upper bound on the bytes of per-edge tensor-product weights materialised at once by the streaming path (edges are
# processed in blocks); additionally capped by a quarter of the free device memory at call time
WEIGHT_BLOCK_BYTES = 2 << 30


def _weight_block_edges(weight_numel_padded, device):
    cap = WEIGHT_BLOCK_BYTES
    try:
        free, _ = torch.cuda.mem_get_info(device)
        cap = min(cap, max(free // 4, 64 << 20))
    except Exception:
        pass
    return max(1024, cap // (4 * weight_numel_padded))


def get_irrep_seq(ns, nv, use_second_order_repr, reduce_pseudoscalars):
    """Same four-stage irreps ladder as models/tensor_layers.py:17-32."""
    tail = f'{nv if reduce_pseudoscalars else ns}x0o'
    if use_second_order_repr:
        steps = [f'{ns}x0e', f'{nv}x1o + {nv}x2e', f'{nv}x1e + {nv}x2o', tail]
    else:
        steps = [f'{ns}x0e', f'{nv}x1o', f'{nv}x1e', tail]
    return [' + '.join(steps[:i + 1]) for i in range(4)]


def irrep_to_size(irrep):
    return irreps_dim(parse_irreps(irrep))


def FCBlock(in_dim, hidden_dim, out_dim, layers, dropout, activation='relu'):
    """Radial MLP with the reference's nn.Sequential index layout (models/layers.py:10-17)."""
    act = ACTIVATIONS[activation]
    assert layers >= 2
    mods = [nn.Linear(in_dim, hidden_dim), act(), nn.Dropout(dropout)]
    for _ in range(layers - 2):
        mods += [nn.Linear(hidden_dim, hidden_dim), act(), nn.Dropout(dropout)]
    mods.append(nn.Linear(hidden_dim, out_dim))
    return nn.Sequential(*mods)


class IrrepsBatchNorm(nn.Module):
    """Parameter container with e3nn.nn.BatchNorm's state_dict layout; eval-mode arithmetic is folded into a
    per-column (scale, shift) pair consumed by the convolution epilogue (ddb200_tpconv_finalize)."""

    def __init__(self, irreps, eps=1e-5):
        super().__init__()
        self.irreps = parse_irreps(irreps)
        self.eps = eps
        n_scalar = sum(m for m, l, p in self.irreps if l == 0 and p == 1)
        n_field = sum(m for m, _, _ in self.irreps)
        self.register_buffer('running_mean', torch.zeros(n_scalar))
        self.register_buffer('running_var', torch.ones(n_field))
        self.weight = nn.Parameter(torch.ones(n_field))
        self.bias = nn.Parameter(torch.zeros(n_scalar))
        rep, sc_col, sc_idx, col, f, s = [], [], [], 0, 0, 0
        for m, l, p in self.irreps:
            d = 2 * l + 1
            for u in range(m):
                rep += [f + u] * d
                if l == 0 and p == 1:
                    sc_col.append(col + u)
                    sc_idx.append(s + u)
            col += m * d
            f += m
            if l == 0 and p == 1:
                s += m
        self.register_buffer('_rep', torch.tensor(rep, dtype=torch.long), persistent=False)
        self.register_buffer('_sc_col', torch.tensor(sc_col, dtype=torch.long), persistent=False)
        self.register_buffer('_sc_idx', torch.tensor(sc_idx, dtype=torch.long), persistent=False)
        self._cache = None

    def fold(self):
        key = (self.weight._version, self.bias._version, self.running_mean._version, self.running_var._version,
               self.weight.device)
        if self._cache is None or self._cache[0] != key:
            with torch.no_grad():
                s_f = self.weight * (self.running_var + self.eps).pow(-0.5)
                scale = s_f[self._rep].contiguous().float()
                shift = torch.zeros_like(scale)
                if self._sc_col.numel():
                    shift[self._sc_col] = self.bias[self._sc_idx] - self.running_mean[self._sc_idx] * scale[self._sc_col]
            self._cache = (key, scale, shift)
        return self._cache[1], self._cache[2]


class _TpSpec(nn.Module):
    """Stands where the reference keeps ``self.tp`` (weight_numel, irreps); holds the kernel tables."""

    def __init__(self, in_irreps, sh_irreps, out_irreps, kind):
        super().__init__()
        self.kind = kind
        self.in_irreps, self.sh_irreps, self.out_irreps = in_irreps, sh_irreps, out_irreps
        shs = parse_irreps(sh_irreps)
        self.vec_capable = shs == [(1, l, (-1) ** l) for l in range(len(shs))] and len(shs) <= 3
        self.table_sh = build_table(in_irreps, sh_irreps, out_irreps, kind, sh_from_vector=False)
        self.table_vec = build_table(in_irreps, sh_irreps, out_irreps, kind, sh_from_vector=True) \
            if self.vec_capable else None
        self.weight_numel = self.table_sh.weight_numel
        self._handles = {}

    def handle(self, from_vec):
        k = bool(from_vec)
        if k not in self._handles:
            self._handles[k] = ops.TpHandle(self.table_vec if k else self.table_sh)
        return self._handles[k]


class TensorProductConvLayer(nn.Module):
    def __init__(self, in_irreps, sh_irreps, out_irreps, n_edge_features, residual=True, batch_norm=True, dropout=0.0,
                 hidden_features=None, faster=False, edge_groups=1, tp_weights_layers=2, activation='relu',
                 depthwise=False):
        super().__init__()
        if depthwise:
            raise NotImplementedError("depthwise_convolution is outside the hot-path scope (SURVEY.md section 8)")
        self.in_irreps, self.out_irreps, self.sh_irreps = in_irreps, out_irreps, sh_irreps
        self.residual, self.edge_groups = residual, edge_groups
        self.out_size = irrep_to_size(out_irreps) if isinstance(out_irreps, str) else irreps_dim(parse_irreps(out_irreps))
        self.depthwise = False
        if hidden_features is None:
            hidden_features = n_edge_features
        self.tp = _TpSpec(in_irreps, sh_irreps, out_irreps, 'faster' if faster else 'fctp')
        if edge_groups == 1:
            self.fc = FCBlock(n_edge_features, hidden_features, self.tp.weight_numel, tp_weights_layers, dropout, activation)
        else:
            self.fc = nn.ModuleList([FCBlock(n_edge_features, hidden_features, self.tp.weight_numel, tp_weights_layers,
                                             dropout, activation) for _ in range(edge_groups)])
        self.batch_norm = IrrepsBatchNorm(out_irreps) if batch_norm else None
        self._wcache = {}
        self._gcache = {}
        self._fcache = {}
        self._pcache = {}

    # -- radial MLP -> per-edge weights in kernel layout ------------------------------------------------------
    def _last_linear(self, fc, table):
        """(weight, bias) of the last Linear, permuted/padded to the kernel's weight-row layout if needed."""
        lin = fc[-1]
        if table.identity_layout:
            return lin.weight, lin.bias
        key = (id(fc), lin.weight._version, lin.bias._version, lin.weight.device)
        hit = self._wcache.get(id(fc))
        if hit is None or hit[0] != key:
            perm = torch.as_tensor(table.w_perm, device=lin.weight.device)
            ok = perm >= 0
            W = lin.weight.new_zeros((perm.numel(), lin.weight.shape[1]))
            b = lin.bias.new_zeros(perm.numel())
            W[ok], b[ok] = lin.weight.detach()[perm[ok]], lin.bias.detach()[perm[ok]]
            hit = (key, W, b)
            self._wcache[id(fc)] = hit
        return hit[1], hit[2]

    def _fused_images(self, fc, table):
        """Operand images of both Linear layers for the one-kernel radial MLP (cached per parameter version)."""
        l1, l2 = fc[0], fc[-1]
        key = (l1.weight._version, l1.bias._version, l2.weight._version, l2.bias._version, l2.weight.device)
        hit = self._fcache.get(id(fc))
        if hit is None or hit[0] != key:
            W2, b2 = self._last_linear(fc, table)
            img1, b1, _ = radial.build_b_images(l1.weight, l1.bias)
            img2, b2p, nt = radial.build_b_images(W2, b2)
            hit = (key, img1, b1, img2, b2p, nt)
            self._fcache[id(fc)] = hit
        return hit[1:]

    def _fused_plan(self, fc, table, k_in, swap_ns=0):
        """Plan of the fully fused kernel for this radial MLP, or None when the shapes are outside its templates.
        ``swap_ns`` > 0: the MLP was trained on ``[ea | node[src] | node[tgt]]`` (ns columns each) while the kernel assembles
        ``[ea | node[tgt] | node[src]]``, so the two node blocks of the first Linear's columns trade places in the plan."""
        if not (fused.ENABLED and self._fused_mlp(fc, k_in) and fused.supported(table, fc[0].out_features, k_in)):
            return None
        lins = [m for m in fc if isinstance(m, nn.Linear)]
        l1, l2 = lins[0], lins[-1]
        key = tuple(v for lin in lins for v in (lin.weight._version, lin.bias._version)) + (l2.weight.device,)
        hit = self._pcache.get((id(fc), swap_ns))
        if hit is None or hit[0] != key:
            w1 = l1.weight
            if swap_ns:
                ne = k_in - 2 * swap_ns
                w1 = torch.cat([w1[:, :ne], w1[:, ne + swap_ns:], w1[:, ne:ne + swap_ns]], 1)
            hidden = [(lin.weight, lin.bias) for lin in lins[1:-1]]
            hit = (key, fused.FusedPlan(table, w1, l1.bias, l2.weight, l2.bias, hidden=hidden))
            self._pcache[(id(fc), swap_ns)] = hit
        return hit[1]

    @staticmethod
    def _fused_mlp(fc, k_in):
        """True if the radial MLP ``fc`` can run inside the fully fused kernel: ``[Linear, ReLU, Dropout] x (L - 1) +
        [Linear]`` (FCBlock with ``tp_weights_layers`` = L >= 2, ReLU), every hidden Linear H x H, H <= fused.MAX_K."""
        mods = list(fc)
        n = (len(mods) + 2) // 3
        if not (radial.USE_TENSOR_CORES and n >= 2 and len(mods) == 3 * n - 2 and k_in <= radial.MAX_K):
            return False
        if not (isinstance(mods[0], nn.Linear) and isinstance(mods[-1], nn.Linear)):
            return False
        H = mods[0].out_features
        if H > fused.MAX_K or mods[-1].in_features != H:
            return False
        for i in range(n - 1):
            lin, act, drop = mods[3 * i:3 * i + 3]
            if not (isinstance(lin, nn.Linear) and isinstance(act, nn.ReLU) and isinstance(drop, nn.Dropout)):
                return False
            if i > 0 and (lin.in_features, lin.out_features) != (H, H):
                return False
        return True

    @staticmethod
    def _fusable(fc, k_in):
        """The host-sized path's one-kernel radial MLP (``ddb200_radial_mlp``): two-layer FCBlocks only."""
        return (radial.USE_TENSOR_CORES and len(fc) == 4 and isinstance(fc[1], nn.ReLU) and isinstance(fc[0], nn.Linear)
                and isinstance(fc[3], nn.Linear) and fc[0].out_features <= radial.MAX_K and k_in <= radial.MAX_K)

    def _edge_weights_fused(self, fc, table, ea, node, ns, tgt32, src32):
        """Per-edge TP weights from the raw pieces: [ea | node[tgt,:ns] | node[src,:ns]] -> Linear -> ReLU -> Linear, all
        inside ddb200_radial_mlp (split-bf16 wgmma GEMMs; no concatenated edge_attr_, no hidden tensor in HBM)."""
        img1, b1, img2, b2p, nt = self._fused_images(fc, table)
        return radial.radial_mlp(ea, node, ns, tgt32, src32, img1, b1, fc[0].out_features, img2, b2p, nt)

    def _edge_weights(self, fc, table, edge_attr):
        """Radial MLP -> per-edge tensor-product weights [E, >= weight_numel_padded] in the kernel's row layout.
        The last (dominant) Linear runs on the Hopper tensor cores (wgmma) as a split-bf16 GEMM (csrc/radial_gemm.cu);
        DDB200_RADIAL_GEMM=cublas selects the plain fp32 library GEMM instead."""
        h = edge_attr
        for m in list(fc)[:-1]:
            h = m(h)
        if radial.USE_TENSOR_CORES and h.shape[1] <= radial.MAX_K and h.shape[0] >= 64:
            lin = fc[-1]
            key = (lin.weight._version, lin.bias._version, lin.weight.device)
            hit = self._gcache.get(id(fc))
            if hit is None or hit[0] != key:
                W, b = self._last_linear(fc, table)
                hit = (key,) + radial.build_b_images(W, b)
                self._gcache[id(fc)] = hit
            return radial.radial_gemm(h.contiguous(), hit[1], hit[2], hit[3])
        W, b = self._last_linear(fc, table)
        return F.linear(h, W, b)

    # -- forward -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, node_attr, edge_index, edge_attr, edge_sh, out_nodes=None, reduce='mean', edge_weight=1.0,
                edge_vec=None, assume_sorted=False, gather_scalars=0, _conv_only=False):
        """Reference signature (models/tensor_layers.py:309) plus optional extensions:
        ``edge_vec`` [E,3]: evaluate the spherical harmonics in-kernel from the edge vectors (``edge_sh`` is ignored);
        ``assume_sorted``: every edge group is already sorted by target node ``edge_index[0]``;
        ``gather_scalars`` = ns > 0: ``edge_attr`` holds only the per-edge part and the radial-MLP kernel appends
        ``node_attr[edge_index[0], :ns]`` and ``node_attr[edge_index[1], :ns]`` itself (models/cg_model.py:342-349)."""
        if self.training:
            raise RuntimeError("diffdock_b200 layers are inference-only: call .eval()")
        if edge_index.shape[1] == 0 and node_attr.shape[0] == 0:
            raise ValueError("No edges and no nodes")
        if not node_attr.is_cuda:
            raise RuntimeError("diffdock_b200.TensorProductConvLayer runs on CUDA tensors only (no CPU fallback)")
        assert reduce in ('mean', 'sum'), "Only 'mean' and 'sum' are supported for reduce"
        _dtype = node_attr.dtype
        x = node_attr.float()
        if x.stride(1) != 1:
            x = x.contiguous()
        n_out = int(out_nodes) if out_nodes else x.shape[0]
        E = edge_index.shape[1]
        scale, shift = self.batch_norm.fold() if (self.batch_norm is not None and not _conv_only) else (None, None)
        residual = self.residual and not _conv_only      # _conv_only: the bare convolution (OldTensorProductConvLayer)
        if E == 0:   # models/tensor_layers.py:314-315: zeros, no BatchNorm, residual still applies
            out = torch.zeros((x.shape[0], self.out_size), dtype=torch.float32, device=x.device)
            if residual:
                out[:, :x.shape[1]] += x
            return out.to(_dtype)

        if self.edge_groups == 1:
            assert isinstance(edge_attr, torch.Tensor), "a single edge group takes a tensor edge_attr"
            groups, fcs = [edge_attr], [self.fc]
        else:
            assert isinstance(edge_attr, list), "This function is only for a list of edge groups"
            groups = edge_attr
            fcs = list(self.fc) if isinstance(self.fc, nn.ModuleList) else [self.fc] * len(groups)
        assert sum(g.shape[0] for g in groups) == E, "Sum of edge_attr_groups must be equal to edge_index.shape[1]"

        from_vec = edge_vec is not None and self.tp.vec_capable
        geo_all = (edge_vec if from_vec else edge_sh).float()
        ew_all = edge_weight if torch.is_tensor(edge_weight) else None
        ew_scalar = 1.0 if torch.is_tensor(edge_weight) else float(edge_weight)
        prepared, s = [], 0
        for ea in groups:
            e = s + ea.shape[0]
            if e > s:
                tgt, src = edge_index[0, s:e], edge_index[1, s:e]
                geo, ew = geo_all[s:e], (ew_all[s:e].reshape(-1) if ew_all is not None else None)
                tgt = tgt.to(torch.int32).contiguous()
                if not assume_sorted:        # CSR order by target: stable device radix sort (ddb200_csr_sort_by_target)
                    tgt, order, _ = ops.csr_sort_by_target(tgt, max(n_out, 1))
                    src, geo, ea = src[order], geo[order], ea[order]
                    if ew is not None:
                        ew = ew[order]
                prepared.append((tgt, src.to(torch.int32).contiguous(), ea, geo.contiguous(), ew))
            else:
                prepared.append(None)
            s = e
        return self._run(x, prepared, fcs, from_vec, ew_scalar, n_out, reduce, gather_scalars, scale, shift,
                         residual=residual, second_order=False).to(_dtype)

    @torch.no_grad()
    def forward_groups(self, node_attr, groups, out_nodes=None, reduce='mean', gather_scalars=0, init=None):
        """Fast internal entry (used by diffdock_b200.CGModel): ``groups`` is a list with one item per radial MLP of this
        layer, each ``(tgt_int32, src_int32, edge_attr, edge_vec, edge_weight | None[, extras])`` already CSR-sorted by
        target, so that no per-layer concatenation / conversion / slicing of the edge arrays is needed.  ``extras`` (dict)
        carries the indirections of the fused kernel - ``n_edges_dev`` (live edge count in device memory, the arrays are
        upper-bound buffers), ``edge_perm``, ``vec_sign``, ``ea_add`` / ``ea_add_idx`` (diffdock_b200/fused.py:fused_conv) -
        and requires a layer shape the fused kernel supports.  A ``None`` entry skips that group's radial MLP;
        ``init = (sum [n_out, D_out], cnt [n_out])`` are accumulators the layer starts from instead of zeros (messages
        computed elsewhere, see ``accumulate_group``)."""
        x = node_attr.float()
        if x.stride(1) != 1:
            x = x.contiguous()
        n_out = int(out_nodes) if out_nodes else x.shape[0]
        scale, shift = self.batch_norm.fold() if self.batch_norm is not None else (None, None)
        fcs = [self.fc] * len(groups) if self.edge_groups == 1 else list(self.fc)
        prepared = [g if (g is not None and g[0].shape[0] > 0) else None for g in groups]
        if all(g is None for g in prepared) and init is None:
            out = torch.zeros((x.shape[0], self.out_size), dtype=torch.float32, device=x.device)
            if self.residual:
                out[:, :x.shape[1]] += x
            return out
        return self._run(x, prepared, fcs, True, 1.0, n_out, reduce, gather_scalars, scale, shift, init=init)

    @torch.no_grad()
    def accumulate_group(self, node_attr, group, group_index, n_out, gather_scalars=0, init=None, swap_gathered=False):
        """Raw accumulators ``(sum [n_out, D_out], cnt [n_out])`` of ONE edge group (radial MLP ``group_index`` of this layer)
        without the mean / BatchNorm / residual epilogue - for messages that are shared by several target blocks (the
        receptor<-receptor messages of the first interaction layer are identical for all poses of a complex) and are added to
        the layer's accumulators through ``forward_groups(..., init=...)``, or that are finalised by the caller.  ``init``:
        accumulators to add to (returned) instead of fresh zeros.  ``swap_gathered``: the radial MLP reads the gathered node's
        scalars before the target's (``[ea | node[src] | node[tgt]]``, models/old_cg_model.py:264-265); fused kernel only."""
        x = node_attr.float()
        if x.stride(1) != 1:
            x = x.contiguous()
        fcs = [self.fc] if self.edge_groups == 1 else list(self.fc)
        fc = fcs[0] if self.edge_groups == 1 else fcs[group_index]
        return self._run(x, [group], [fc], True, 1.0, int(n_out), 'sum', gather_scalars, None, None, init=init,
                         finalize=False, swap_gathered=swap_gathered)

    def fused_capable(self, k_edge, gather_scalars):
        """True if every radial MLP of this layer runs on the fully fused kernel for ``k_edge`` per-edge attribute columns
        (+ 2 x ``gather_scalars`` node scalars) with in-kernel spherical harmonics, through ``forward_groups`` (layers with
        l = 2 blocks: through the grouped entry points only, see ``_run``)."""
        if not self.tp.vec_capable:
            return False
        table = self.tp.table_vec
        fcs = [self.fc] if self.edge_groups == 1 else list(self.fc)
        k_in = k_edge + 2 * gather_scalars
        return all(fused.ENABLED and self._fused_mlp(fc, k_in) and fused.supported(table, fc[0].out_features, k_in)
                   for fc in fcs)

    def _run(self, x, prepared, fcs, from_vec, ew_scalar, n_out, reduce, gather_scalars, scale, shift, residual=None,
             init=None, finalize=True, swap_gathered=False, second_order=True):
        """``second_order``: layers with l = 2 blocks may take the fused kernel's second-order instantiation.  Only the
        grouped entry points (``forward_groups`` / ``accumulate_group``, the models' convolution stacks) allow it; the
        reference-signature ``forward`` keeps such layers on the streaming kernel, as it ran them before that
        instantiation existed."""
        handle = self.tp.handle(from_vec)
        table = handle.table
        if init is not None:
            sum_buf, cnt_buf = init
            assert tuple(sum_buf.shape) == (n_out, self.out_size) and sum_buf.is_contiguous() and cnt_buf.shape[0] == n_out
        else:       # int64 fixed point under torch.use_deterministic_algorithms(True) (ops.new_accumulators)
            sum_buf, cnt_buf = ops.new_accumulators(n_out, self.out_size, x.device)
        blk = None
        for item, fc in zip(prepared, fcs):
            if item is None:
                continue
            tgt32, src32, ea, geo, ew = item[:5]
            extras = item[5] if len(item) > 5 else None
            n_e = tgt32.shape[0]
            k_in = ea.shape[1] + 2 * gather_scalars
            plan = self._fused_plan(fc, table, k_in, gather_scalars if swap_gathered else 0) \
                if (from_vec and ew_scalar == 1.0 and (n_e >= 64 or extras is not None)
                    and (second_order or not fused.second_order(table))) else None
            if swap_gathered and plan is None:
                raise RuntimeError("swapped node scalars (swap_gathered) need a fused-kernel layer shape "
                                   "(TensorProductConvLayer.fused_capable)")
            if plan is not None:      # radial MLP + tensor product + scatter in one kernel, no per-edge weights in HBM
                fused.fused_conv(plan, ea.float(), x, gather_scalars, tgt32, src32, x, geo.float(), sum_buf, cnt_buf,
                                 edge_weight=ew.float().contiguous() if ew is not None else None, **(extras or {}))
                continue
            if extras is not None:
                raise RuntimeError("edge groups with device-side counts / indirections need a fused-kernel layer shape "
                                   "(TensorProductConvLayer.fused_capable)")
            mlp_fused = self._fusable(fc, k_in) and n_e >= 64
            if blk is None:
                blk = _weight_block_edges(table.weight_numel_padded, x.device)
            if gather_scalars and not mlp_fused:     # library path needs the concatenated attributes
                ea = torch.cat([ea, x[tgt32.long(), :gather_scalars], x[src32.long(), :gather_scalars]], -1)
            for b0 in range(0, n_e, blk):
                b1 = min(n_e, b0 + blk)
                if mlp_fused:
                    w = self._edge_weights_fused(fc, table, ea[b0:b1].float(), x, gather_scalars, tgt32[b0:b1],
                                                 src32[b0:b1])
                else:
                    w = self._edge_weights(fc, table, ea[b0:b1].float())
                if ew_scalar != 1.0:
                    w = w * ew_scalar
                ops.tpconv_accumulate(handle, x, src32[b0:b1], tgt32[b0:b1], geo[b0:b1], w, sum_buf, cnt_buf,
                                      edge_weight=ew[b0:b1] if ew is not None else None, count_node_bytes=b0 == 0)
                del w
        if not finalize:
            return sum_buf, cnt_buf
        res = x if (self.residual if residual is None else residual) else None
        return ops.tpconv_finalize(sum_buf, cnt_buf, reduce == 'mean', scale, shift, res)


class OldTensorProductConvLayer(TensorProductConvLayer):
    """Drop-in for models/tensor_layers.py:338-380 (the confidence model's layer): one radial MLP, same kernels as the new
    layer.  The reference's 100 000-edge chunking only bounds memory (all chunks share the MLP) and is not reproduced;
    the residual is added BEFORE the BatchNorm (:371-376), unlike the new layer."""

    def __init__(self, in_irreps, sh_irreps, out_irreps, n_edge_features, residual=True, batch_norm=True, dropout=0.0,
                 hidden_features=None):
        super().__init__(in_irreps, sh_irreps, out_irreps, n_edge_features, residual=residual, batch_norm=batch_norm,
                         dropout=dropout, hidden_features=hidden_features, faster=False, edge_groups=1,
                         tp_weights_layers=2, activation='relu')

    @torch.no_grad()
    def forward(self, node_attr, edge_index, edge_attr, edge_sh, out_nodes=None, reduce='mean', edge_weight=1.0,
                edge_vec=None, assume_sorted=False, gather_scalars=0):
        if edge_index.shape[1] == 0:
            # No edge at all (e.g. a pose without any receptor atom within 5 A): the reference divides the edges into zero
            # chunks and raises (np.array_split, models/tensor_layers.py:362-365).  Here the convolution contributes zeros
            # to its out_nodes rows and the usual epilogue (residual, BatchNorm) follows.
            n_out = int(out_nodes) if out_nodes else node_attr.shape[0]
            out = node_attr.new_zeros((n_out, self.out_size), dtype=torch.float32)
            if self.residual:
                out = out + F.pad(node_attr.float(), (0, out.shape[-1] - node_attr.shape[-1]))
            if self.batch_norm is not None:
                scale, shift = self.batch_norm.fold()
                out = out * scale + shift
            return out.to(node_attr.dtype)
        if not self.residual:
            return super().forward(node_attr, edge_index, edge_attr, edge_sh, out_nodes, reduce, edge_weight,
                                   edge_vec=edge_vec, assume_sorted=assume_sorted, gather_scalars=gather_scalars)
        bn = self.batch_norm                                                      # conv only, then residual -> BatchNorm
        out = super().forward(node_attr, edge_index, edge_attr, edge_sh, out_nodes, reduce, edge_weight,
                              edge_vec=edge_vec, assume_sorted=assume_sorted, gather_scalars=gather_scalars,
                              _conv_only=True)
        out = out + F.pad(node_attr, (0, out.shape[-1] - node_attr.shape[-1]))
        if bn is not None:
            scale, shift = bn.fold()
            out = out * scale + shift
        return out.to(node_attr.dtype)
