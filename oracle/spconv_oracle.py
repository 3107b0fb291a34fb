"""oracle/spconv_oracle.py -- CPU restatement of the sparse convolutions the reference delegates to spconv 2.x.
TEST INFRASTRUCTURE ONLY (same import rule as the rest of oracle/).

PARITY UNPINNED by the reference: spconv (PyPI `spconv-cu102`, "2.1" per README.md:20 / docs/installation.md:27) is
not vendored under /root/reference and not installed here, and the reference has no test that pins results at this
boundary (SURVEY.md 4, 8c). The semantics below restate spconv 2.x as used by the reference call sites
(softgroup/model/blocks.py:31-41,50-70,96-129):
  * indices int32 [M,4] = (batch, d0, d1, d2); weight [out, k0, k1, k2, in] (tools/convert_checkpoint.py:17-19)
  * cross-correlation orientation, identical to F.conv3d with the weight permuted to [out, in, k0, k1, k2]
  * SubMConv3d k3 p1: output sites = input sites, absent neighbours contribute 0
  * SparseConv3d k2 s2 p0: out_shape = floor((D-2)/2)+1; parent = coord // 2; inputs whose parent >= out_shape (max plane
    of an odd dim) are dropped; output sites = distinct parents (here numbered by first occurrence in input order --
    the numbering is unobservable through the U-Net because the paired inverse conv restores the input order)
  * SparseInverseConv3d k2: out[child] = W[:, o, :] . in[parent], o = child - 2*parent, output sites/order = the paired
    conv's input sites
and are cross-checked against dense torch F.conv3d / F.conv_transpose3d on small grids in tests/test_spconv_oracle.py,
which is what anchors them.
numpy, float32 storage, float64 accumulation option for tight comparisons.
"""
import numpy as np


def _pack(idx):
    idx = idx.astype(np.int64)
    return ((idx[:, 0] << 48) | ((idx[:, 1] + 1) << 32) | ((idx[:, 2] + 1) << 16) | (idx[:, 3] + 1))


def _lookup(keys_sorted, order, q):
    if len(keys_sorted) == 0:  # e.g. a down2 level without parents
        return np.full(len(q), -1, np.int64)
    pos = np.searchsorted(keys_sorted, q)
    pos = np.clip(pos, 0, len(keys_sorted) - 1)
    hit = keys_sorted[pos] == q
    return np.where(hit, order[pos], -1)


def subm_map(indices):
    """int32 [27, M]: map[k][j] = row of indices[j] + (k0-1, k1-1, k2-1) or -1."""
    M = indices.shape[0]
    keys = _pack(indices)
    order = np.argsort(keys, kind='stable')
    ks = keys[order]
    out = np.full((27, M), -1, np.int32)
    for k in range(27):
        d = np.array([0, k // 9 - 1, (k // 3) % 3 - 1, k % 3 - 1])
        out[k] = _lookup(ks, order, _pack(indices + d))
    return out


def down_map(indices, spatial_shape):
    """-> out_indices int32 [Mout,4], map int32 [8,Mout], inv_map int32 [8,M], out_shape."""
    M = indices.shape[0]
    out_shape = [int(s) // 2 for s in spatial_shape]  # floor((D-2)/2)+1
    par = indices.copy()
    par[:, 1:] = indices[:, 1:] >> 1
    valid = np.all(par[:, 1:] < np.array(out_shape), axis=1)
    keys = _pack(par)
    keys_v = np.where(valid, keys, -1)
    uniq, first = np.unique(keys_v[valid], return_index=True)
    vrows = np.where(valid)[0]
    first_rows = np.sort(vrows[first])  # first occurrence order
    out_indices = par[first_rows].astype(np.int32)
    okeys = _pack(out_indices)
    oorder = np.argsort(okeys, kind='stable')
    pid = _lookup(okeys[oorder], oorder, keys)
    pid = np.where(valid, pid, -1)
    Mout = out_indices.shape[0]
    k = ((indices[:, 1] & 1) * 2 + (indices[:, 2] & 1)) * 2 + (indices[:, 3] & 1)
    mp = np.full((8, Mout), -1, np.int32)
    inv = np.full((8, M), -1, np.int32)
    rows = np.arange(M)
    mp[k[valid], pid[valid]] = rows[valid]
    inv[k[valid], rows[valid]] = pid[valid]
    return out_indices, mp, inv, out_shape


def conv_from_map(feats, mp, weight, acc64=False):
    """out[j] = sum_k W[:, k, :] . feats[map[k][j]]   (weight [out, K..., in] flattened over the kernel dims)."""
    Cout, Cin = weight.shape[0], weight.shape[-1]
    W = weight.reshape(Cout, -1, Cin)
    K = W.shape[1]
    assert mp.shape[0] == K
    dt = np.float64 if acc64 else np.float32
    out = np.zeros((mp.shape[1], Cout), dt)
    f = feats.astype(dt)
    for k in range(K):
        sel = mp[k] >= 0
        if sel.any():
            out[sel] += f[mp[k][sel]] @ W[:, k, :].astype(dt).T
    return out.astype(np.float32)


def subm_conv3d(feats, indices, weight, acc64=False):
    return conv_from_map(feats, subm_map(indices), weight, acc64)


def sparse_conv3d_k2s2(feats, indices, spatial_shape, weight, acc64=False):
    out_indices, mp, inv, out_shape = down_map(indices, spatial_shape)
    return conv_from_map(feats, mp, weight, acc64), out_indices, inv, out_shape


def inverse_conv3d_k2(feats_coarse, inv_map, weight, acc64=False):
    return conv_from_map(feats_coarse, inv_map, weight, acc64)


# ---------------------------------------------------------------------------------------------------------
# Whole U-Net restatement (softgroup/model/blocks.py:44-143) on top of the functions above, for parity tests of
# the backbone. `sd` is a state_dict-like {name: numpy array} using the reference's parameter names.
# ---------------------------------------------------------------------------------------------------------
def _bn_relu(x, sd, prefix, eps=1e-4, acc64=False):
    dt = np.float64 if acc64 else np.float32
    w, b = sd[prefix + '.weight'].astype(dt), sd[prefix + '.bias'].astype(dt)
    m, v = sd[prefix + '.running_mean'].astype(dt), sd[prefix + '.running_var'].astype(dt)
    y = (x.astype(dt) - m) / np.sqrt(v + dt(eps)) * w + b
    return np.maximum(y, 0).astype(np.float32)


def residual_block(x, smap, sd, prefix, acc64=False):
    """blocks.py:44-79. conv_branch = [BN, ReLU, SubM, BN, ReLU, SubM]; i_branch = identity or 1x1."""
    if (prefix + '.i_branch.0.weight') in sd:
        W = sd[prefix + '.i_branch.0.weight']
        ident = conv_from_map(x, np.arange(x.shape[0], dtype=np.int32)[None], W, acc64)
    else:
        ident = x
    h = _bn_relu(x, sd, prefix + '.conv_branch.0', acc64=acc64)
    h = conv_from_map(h, smap, sd[prefix + '.conv_branch.2.weight'], acc64)
    h = _bn_relu(h, sd, prefix + '.conv_branch.3', acc64=acc64)
    h = conv_from_map(h, smap, sd[prefix + '.conv_branch.5.weight'], acc64)
    return h + ident


def ublock(x, indices, spatial_shape, sd, prefix, nplanes, acc64=False):
    """blocks.py:82-143."""
    smap = subm_map(indices)
    for i in range(2):
        x = residual_block(x, smap, sd, '%s.blocks.block%d' % (prefix, i), acc64)
    if len(nplanes) > 1:
        ident = x
        h = _bn_relu(x, sd, prefix + '.conv.0', acc64=acc64)
        out_idx, mp, inv, out_shape = down_map(indices, spatial_shape)
        h = conv_from_map(h, mp, sd[prefix + '.conv.2.weight'], acc64)
        h = ublock(h, out_idx, out_shape, sd, prefix + '.u', nplanes[1:], acc64)
        h = _bn_relu(h, sd, prefix + '.deconv.0', acc64=acc64)
        h = conv_from_map(h, inv, sd[prefix + '.deconv.2.weight'], acc64)
        x = np.concatenate([ident, h], 1)
        for i in range(2):
            x = residual_block(x, smap, sd, '%s.blocks_tail.block%d' % (prefix, i), acc64)
    return x


def backbone(voxel_feats, voxel_indices, spatial_shape, sd, channels, num_blocks, acc64=False):
    """softgroup/model/softgroup.py:363-378 up to output_layer (returns per-voxel features)."""
    smap = subm_map(voxel_indices)
    x = conv_from_map(voxel_feats, smap, sd['input_conv.0.weight'], acc64)
    x = ublock(x, voxel_indices, spatial_shape, sd, 'unet', [channels * (i + 1) for i in range(num_blocks)], acc64)
    return _bn_relu(x, sd, 'output_layer.0', acc64=acc64)
