"""The cases tests/test_gpu_hash_edges.py runs for the two GPU hash tables -- point-to-voxel hashing (voxelize.cu:
sgb_voxelize_idx_count / _fill) and the sparse-convolution rulebooks (spconv.cu: sgb_rulebook_subm3,
sgb_rulebook_down2_count / _fill) -- next to numpy restatements of their key packing, hash and capacity rules and the
constants the cases must reach. tests/test_hash_coverage.py checks on the CPU that the table reaches every edge, and that
the constants below still match the sources."""
import collections

import numpy as np

# ---- constants of softgroup_b200/csrc -------------------------------------------------------------------------------
EMPTY_KEY = 0xFFFFFFFFFFFFFFFF  # common.cuh kEmptyKey: the marker of an empty slot
HASH_SHIFTS = (33, 33, 33)  # common.cuh hash64: k ^= k >> s, k *= m, ... (the murmur3 finaliser)
HASH_MULS = (0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53)
# voxelize.cu pack_key: [batch:16][x+32768:16][y+32768:16][z+32768:16]; accepted b in [0, 65535], xyz in [-32768, 32767]
VOX_B = (0, 65535)
VOX_XYZ = (-32768, 32767)
VOX_XYZ_BIAS = 32768
# spconv.cu vkey: [b:16][x+1:16][y+1:16][z+1:16]; idx_ok accepts b in [0, 65535], xyz in [0, 32766]
RB_B = (0, 65535)
RB_XYZ = (0, 32766)
RB_XYZ_BIAS = 1
SORT_INSERTION_MAX = 24  # vox_sort_rows_kernel: rows of <= 24 entries are insertion-sorted by their own lane
SORT_WARP_MAX = 32 * 32  # rows of <= 1024 entries (nchunk <= 32) are rank-sorted by the warp, longer ones by lane 0
SCAN_TILE = 512 * 8  # core.cu kScanTile: exclusive_scan_i32 takes 1 level up to one tile, 2 up to SCAN_TILE**2, then 3
ROW_LENGTHS = (1, 2, 24, 25, 32, 33, 1024, 1025, 3000)


# ---- numpy restatements ---------------------------------------------------------------------------------------------
def hash64(keys):
    """common.cuh hash64 of uint64 keys -> uint32."""
    k = np.array(keys, np.uint64, ndmin=1)
    for i, s in enumerate(HASH_SHIFTS):
        k ^= k >> np.uint64(s)
        if i < len(HASH_MULS):
            k *= np.uint64(HASH_MULS[i])  # wraps mod 2^64, like the device multiply
    return (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def pow2_at_least(x):
    c = 1
    while c < x:
        c <<= 1
    return c


def vox_cap(n):
    """voxelize.cu vox_cap: table slots for n points."""
    return pow2_at_least(max(n, 1) * 2)


def rb_cap(m):
    """spconv.cu rb_cap: table slots for m rows."""
    return pow2_at_least(max(m, 1) * 2)


def home(keys, cap):
    """First slot hash_insert / hash_find probe for each key."""
    return (hash64(keys) & np.uint32(cap - 1)).astype(np.int64)


def _pack16(fields):
    out = np.zeros(len(fields[0]), np.uint64)
    for f in fields:
        out = (out << np.uint64(16)) | (np.asarray(f, np.int64) & 0xFFFF).astype(np.uint64)
    return out


def pack_key(coords, ncol=4):
    """voxelize.cu pack_key of int64 coords [N, ncol] -> (uint64 keys [N], accepted [N])."""
    c = np.asarray(coords, np.int64).reshape(-1, ncol)
    b = c[:, 0] if ncol == 4 else np.zeros(len(c), np.int64)
    xyz = c[:, ncol - 3:]
    ok = (b >= VOX_B[0]) & (b <= VOX_B[1]) & ((xyz >= VOX_XYZ[0]) & (xyz <= VOX_XYZ[1])).all(1)
    return _pack16([b] + [xyz[:, j] + VOX_XYZ_BIAS for j in range(3)]), ok


def unpack_key(keys):
    """Inverse of pack_key (ncol 4): every 64-bit value is the key of exactly one accepted point."""
    k = np.asarray(keys, np.uint64)
    f = [((k >> np.uint64(s)) & np.uint64(0xFFFF)).astype(np.int64) for s in (48, 32, 16, 0)]
    return np.stack([f[0], f[1] - VOX_XYZ_BIAS, f[2] - VOX_XYZ_BIAS, f[3] - VOX_XYZ_BIAS], 1)


def vkey(idx):
    """spconv.cu vkey of int [M, 4] (b, x, y, z) -> uint64."""
    c = np.asarray(idx, np.int64).reshape(-1, 4)
    return _pack16([c[:, 0]] + [c[:, j] + RB_XYZ_BIAS for j in (1, 2, 3)])


def idx_ok(idx):
    """spconv.cu idx_ok: rows the rulebooks accept."""
    c = np.asarray(idx, np.int64).reshape(-1, 4)
    return (c[:, 0] >= RB_B[0]) & (c[:, 0] <= RB_B[1]) & ((c[:, 1:] >= RB_XYZ[0]) & (c[:, 1:] <= RB_XYZ[1])).all(1)


def occupied(homes, cap):
    """Slots a linear-probing table of `cap` slots holds once one key per entry of `homes` is in it. The set does not
    depend on the insertion order."""
    load = np.bincount(np.asarray(homes, np.int64), minlength=cap)
    occ = np.zeros(cap, bool)
    carry = 0
    for s in range(cap):
        carry += int(load[s])
        if carry:
            occ[s] = True
            carry -= 1
    s = 0
    while carry:  # the keys pushed past slot cap - 1 continue at slot 0
        if not occ[s]:
            occ[s] = True
            carry -= 1
        s += 1
    return occ


def chain_lengths(homes, cap):
    """Per key, the probe chain a lookup walks from its home: the occupied slots from there up to the first empty one."""
    occ = occupied(homes, cap)
    run = np.zeros(cap, np.int64)
    nxt = 0
    for s in range(2 * cap - 1, -1, -1):  # two laps, so runs that wrap past slot cap - 1 are counted in full
        nxt = nxt + 1 if occ[s % cap] else 0
        run[s % cap] = nxt
    return run[np.asarray(homes, np.int64)]


def scan_levels(n):
    """Levels of exclusive_scan_i32 over n elements (tiles of SCAN_TILE, then a scan of the tile sums, ...)."""
    lv = 1
    while n > SCAN_TILE:
        n = (n + SCAN_TILE - 1) // SCAN_TILE
        lv += 1
    return lv


# ---- voxelize cases -------------------------------------------------------------------------------------------------
# Every case is int64 coords [N, ncol] from a seeded generator. Points are shuffled, so the duplicates of a voxel land
# in different warps and blocks. Modes 1-4 run on every case; mode 0 ('unique') only on input without duplicates.
def _expand(rng, rows, reps):
    pts = np.repeat(np.asarray(rows, np.int64), reps, axis=0)
    return pts[rng.permutation(len(pts))]


def _keys_with_homes(rng, cap, slots, count, gen=None):
    """`count` distinct keys, none the empty marker, whose home slot at `cap` is in `slots`. gen(rng, n) draws candidate
    keys (default: any 64-bit value, i.e. any accepted voxelize point)."""
    gen = gen or (lambda r, n: r.randint(0, 1 << 62, n, dtype=np.uint64) * np.uint64(4) + r.randint(0, 4, n).astype(np.uint64))
    found = np.zeros(0, np.uint64)
    while len(found) < count:
        k = gen(rng, 1 << 21)
        k = k[np.isin(home(k, cap), slots) & (k != np.uint64(EMPTY_KEY))]
        found = np.unique(np.concatenate([found, k]))
    return found[rng.permutation(len(found))[:count]]


def _corners(seed=0):
    rng = np.random.RandomState(seed)
    v = (VOX_XYZ[0], -1, 0, VOX_XYZ[1])
    rows = np.array([(b, x, y, z) for b in VOX_B for x in v for y in v for z in v], np.int64)
    return _expand(rng, rows, rng.randint(1, 4, len(rows)))


SENTINEL_POINT = (VOX_B[1], VOX_XYZ[1], VOX_XYZ[1], VOX_XYZ[1])  # packs to the empty marker
SENTINEL_PARTNER = (44, 47, 0, 3)  # shares the sentinel's home slot in a table of vox_cap(2) = 4 slots


def _sentinel_merge():
    return np.array([SENTINEL_POINT, SENTINEL_PARTNER], np.int64)


SENTINEL_CROWD_N = 4000


def _sentinel_crowd(seed=1):
    """The sentinel point 40 times across the blocks, 80 keys sharing its home slot at vox_cap(4000) (3 points each),
    and 3720 other random voxels."""
    rng = np.random.RandomState(seed)
    cap = vox_cap(SENTINEL_CROWD_N)
    crowd = unpack_key(_keys_with_homes(rng, cap, home([EMPTY_KEY], cap), 80))
    other = unpack_key(_keys_with_homes(rng, cap, np.arange(cap), SENTINEL_CROWD_N - 40 - 240))
    rows = np.concatenate([[SENTINEL_POINT], crowd, other])
    reps = np.concatenate([[40], np.full(len(crowd), 3), np.ones(len(other), np.int64)])
    return _expand(rng, rows, reps)


def _sentinel_ncol3(seed=2):
    rng = np.random.RandomState(seed)
    rows = np.array([SENTINEL_POINT[1:], (VOX_XYZ[1], VOX_XYZ[1], VOX_XYZ[1] - 1), (-1, -1, -1), (0, 0, 0)], np.int64)
    return _expand(rng, rows, [5, 2, 3, 1])


def _batch_isolation(seed=3):
    rng = np.random.RandomState(seed)
    xyz = rng.randint(-40, 40, (300, 3))
    rows = np.concatenate([np.concatenate([np.full((300, 1), b), xyz], 1) for b in (0, 1, VOX_B[1])])
    return _expand(rng, rows, rng.randint(1, 3, len(rows)))


WRAP_DISTINCT = 2000


def _vox_wrap_probe(seed=4):
    """2000 distinct voxels whose home slots are the last 8 of vox_cap(3000); half of them have a second point."""
    rng = np.random.RandomState(seed)
    cap = vox_cap(WRAP_DISTINCT * 3 // 2)
    rows = unpack_key(_keys_with_homes(rng, cap, np.arange(cap - 8, cap), WRAP_DISTINCT))
    return _expand(rng, rows, np.repeat([2, 1], WRAP_DISTINCT // 2))


def _row_lengths(seed=5):
    """Voxels of exactly 1, 2, 24, 25, 32, 33, 1024, 1025 and 3000 points, three of each, and 37 one-point voxels: the
    long rows come first in voxel-id order, so warp 0 holds several of them next to short rows."""
    rng = np.random.RandomState(seed)
    n = 3 * len(ROW_LENGTHS) + 37
    k = rng.choice(3 * 200 ** 3, n, replace=False)
    rows = np.stack([k // 200 ** 3, (k // 40000) % 200 - 100, (k // 200) % 200 - 100, k % 200 - 100], 1)
    reps = np.concatenate([np.repeat(ROW_LENGTHS, 3), np.ones(37, np.int64)])
    return _expand(rng, rows, reps)


def _size(n, unique, seed):
    """n points; unique: n distinct voxels, else about a third of the points repeat a voxel."""
    rng = np.random.RandomState(seed)
    nv = n if unique else max(1, (2 * n) // 3)
    keys = np.unique(rng.randint(0, 1 << 30, 2 * nv + 8))
    keys = keys[rng.permutation(len(keys))[:nv]]
    rows = np.stack([keys >> 24, (keys >> 16 & 0xFF) - 128, (keys >> 8 & 0xFF) - 128, (keys & 0xFF) - 128], 1)
    pts = np.concatenate([rows, rows[rng.randint(0, nv, n - nv)]])
    return pts[rng.permutation(n)].astype(np.int64)


THREE_LEVEL_N = SCAN_TILE * SCAN_TILE + 1


def _three_level_scan(seed=6):
    """16,777,217 distinct voxels: batch i >> 16, x and y the next bytes, z spread; shuffled."""
    i = np.arange(THREE_LEVEL_N, dtype=np.int64)
    pts = np.stack([i >> 16, ((i >> 8) & 0xFF) - 128, (i & 0xFF) - 128, (i * 7919) % 4001 - 2000], 1)
    return pts[np.random.RandomState(seed).permutation(THREE_LEVEL_N)]


VoxCase = collections.namedtuple('VoxCase', 'name make ncol unique')
VOX_CASES = [
    VoxCase('corners', _corners, 4, False),
    VoxCase('sentinel_merge', _sentinel_merge, 4, True),
    VoxCase('sentinel_crowd', _sentinel_crowd, 4, False),
    VoxCase('sentinel_ncol3', _sentinel_ncol3, 3, False),
    VoxCase('batch_isolation', _batch_isolation, 4, False),
    VoxCase('wrap_probe', _vox_wrap_probe, 4, False),
    VoxCase('row_lengths', _row_lengths, 4, False),
    VoxCase('size_1', lambda: _size(1, True, 10), 4, True),
    VoxCase('size_2', lambda: _size(2, False, 11), 4, False),
    VoxCase('size_4096', lambda: _size(4096, True, 12), 4, True),
    VoxCase('size_4097', lambda: _size(4097, False, 13), 4, False),
    VoxCase('size_65536', lambda: _size(65536, False, 14), 4, False),
    VoxCase('size_65537', lambda: _size(65537, True, 15), 4, True),
    VoxCase('three_level_scan', _three_level_scan, 4, True),
]
LARGE_VOX = ('three_level_scan', )  # too large for the host-path comparison on the CPU


def vox_case(name):
    return [c for c in VOX_CASES if c.name == name][0]


def vox_modes(case):
    return (0, 1, 2, 3, 4) if case.unique else (1, 2, 3, 4)


# Values just outside the accepted range of each field, and one beyond int32 (the host path and the reference narrow
# it to 3; the GPU path rejects it).
VOX_FIELDS = ('b', 'x', 'y', 'z')
VOX_OUT_OF_RANGE = [('b', VOX_B[0] - 1), ('b', VOX_B[1] + 1), ('b', (1 << 32) + 3)] + \
    [(f, v) for f in 'xyz' for v in (VOX_XYZ[0] - 1, VOX_XYZ[1] + 1, (1 << 32) + 3)] + [('z', 40000)]


def vox_out_of_range(field, value, seed=7):
    """300 in-range points (some repeated) with one point whose `field` is `value`, at index 123."""
    pts = _size(300, False, seed)
    pts[123, VOX_FIELDS.index(field)] = value
    return pts


# ---- rulebook cases -------------------------------------------------------------------------------------------------
# Every case is int32 indices [M, 4] (b, x, y, z) with unique rows, and the spatial shape the down2 rulebook is built
# with. 'subm': the case also runs through the subm3 rulebook (the 16.8M-row case only runs down2).
def _unique_rows(rng, parts):
    rows = np.unique(np.concatenate(parts).astype(np.int64), axis=0)
    return rows[rng.permutation(len(rows))].astype(np.int32)


def _block(b, lo, n=3):
    r = np.arange(n)
    g = np.stack(np.meshgrid(r, r, r, indexing='ij'), -1).reshape(-1, 3)
    return np.concatenate([np.full((len(g), 1), b), g + np.asarray(lo)], 1)


RB_MAX_LO = RB_XYZ[1] - 2  # 32764: the block 32764..32766 ends on the last accepted coordinate


def _rb_corners(seed=20):
    rng = np.random.RandomState(seed)
    ends = (0, RB_MAX_LO)
    return _unique_rows(rng, [_block(b, (x, y, z)) for b in RB_B for x in ends for y in ends for z in ends])


def _rb_batch_isolation(seed=21):
    rng = np.random.RandomState(seed)
    xyz = np.unique(rng.randint(0, 16, (900, 3)), axis=0)
    return _unique_rows(rng, [np.concatenate([np.full((len(xyz), 1), b), xyz], 1) for b in (0, 1, RB_B[1])])


def _rb_gen(r, n):
    rows = np.concatenate([r.randint(0, RB_B[1] + 1, (n, 1)), r.randint(0, RB_XYZ[1] + 1, (n, 3))], 1)
    return vkey(rows)


def _rb_unvkey(keys):
    k = np.asarray(keys, np.uint64)
    f = [((k >> np.uint64(s)) & np.uint64(0xFFFF)).astype(np.int64) for s in (48, 32, 16, 0)]
    return np.stack([f[0], f[1] - RB_XYZ_BIAS, f[2] - RB_XYZ_BIAS, f[3] - RB_XYZ_BIAS], 1)


def _rb_wrap_probe(seed=22):
    """2000 rows whose home slots are the last 8 of rb_cap(2000)."""
    rng = np.random.RandomState(seed)
    cap = rb_cap(WRAP_DISTINCT)
    keys = _keys_with_homes(rng, cap, np.arange(cap - 8, cap), WRAP_DISTINCT, gen=_rb_gen)
    return _rb_unvkey(keys).astype(np.int32)


def _dense(shape, b=2, density=0.4, seed=23):
    rng = np.random.RandomState(seed)
    rows = []
    for bi in range(b):
        occ = np.argwhere(rng.rand(*shape) < density)
        rows.append(np.concatenate([np.full((len(occ), 1), bi), occ], 1))
    return _unique_rows(rng, rows)


def _children(seed=24):
    """Parents of a 16^3 grid (shape 32^3) with all 8 children, with 1 child, and parents whose children are all at the
    end of the row order (their first child comes late, so their id is high)."""
    rng = np.random.RandomState(seed)
    par = np.unique(rng.randint(0, 16, (600, 3)), axis=0)
    par = par[rng.permutation(len(par))]
    full, one, late = par[:150], par[150:300], par[300:380]
    off = np.array([(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)])
    kids_full = (2 * full[:, None] + off[None]).reshape(-1, 3)
    kids_one = 2 * one + off[rng.randint(0, 8, len(one))]
    kids_late = (2 * late[:, None] + off[None, rng.permutation(8)[:3]]).reshape(-1, 3)
    early = np.concatenate([kids_full, kids_one])
    early = early[rng.permutation(len(early))]
    late_rows = kids_late[rng.permutation(len(kids_late))]
    rows = np.concatenate([early, late_rows])
    return np.concatenate([np.zeros((len(rows), 1), np.int64), rows], 1).astype(np.int32)


def _rb_size(m, seed):
    rng = np.random.RandomState(seed)
    k = rng.choice(2 * 64 ** 3, m, replace=False)
    return np.stack([k >> 18, (k >> 12) & 63, (k >> 6) & 63, k & 63], 1).astype(np.int32)


RB_THREE_LEVEL_M = SCAN_TILE * SCAN_TILE + 1


def _rb_three_level(seed=25):
    """16,777,217 rows: 64 full 64^3 batches and one more row, shuffled."""
    i = np.arange(RB_THREE_LEVEL_M, dtype=np.int64)
    rows = np.stack([i >> 18, (i >> 12) & 63, (i >> 6) & 63, i & 63], 1).astype(np.int32)
    return rows[np.random.RandomState(seed).permutation(RB_THREE_LEVEL_M)]


RbCase = collections.namedtuple('RbCase', 'name make shape subm')
FULL_SHAPE = (RB_XYZ[1] + 1, ) * 3  # 32767: the parent 16383 of coordinate 32766 is dropped
RB_CASES = [
    RbCase('corners', _rb_corners, FULL_SHAPE, True),
    RbCase('batch_isolation', _rb_batch_isolation, (16, 16, 16), True),
    RbCase('wrap_probe', _rb_wrap_probe, FULL_SHAPE, True),
    RbCase('odd_x', lambda: _dense((9, 8, 8), seed=30), (9, 8, 8), True),
    RbCase('odd_y', lambda: _dense((8, 9, 8), seed=31), (8, 9, 8), True),
    RbCase('odd_z', lambda: _dense((8, 8, 9), seed=32), (8, 8, 9), True),
    RbCase('d1_axis', lambda: _dense((1, 8, 8), seed=33), (1, 8, 8), True),
    RbCase('d2_axis', lambda: _dense((6, 2, 5), seed=34), (6, 2, 5), True),
    RbCase('children', _children, (32, 32, 32), True),
    RbCase('size_1', lambda: _rb_size(1, 40), (64, 64, 64), True),
    RbCase('size_4096', lambda: _rb_size(4096, 41), (64, 64, 64), True),
    RbCase('size_4097', lambda: _rb_size(4097, 42), (64, 64, 64), True),
    RbCase('three_level_scan', _rb_three_level, (64, 64, 64), False),
]


def rb_case(name):
    return [c for c in RB_CASES if c.name == name][0]


# Rows the rulebooks reject: just outside each field, and the row whose (+1, +1, +1) neighbour packs to the empty
# marker. Each goes into a set of accepted rows holding the neighbours it would alias under the 16-bit masking.
RB_OUT_OF_RANGE = [(-1, 5, 5, 5), (RB_B[1] + 1, 5, 5, 5)] + \
    [(0, ) + tuple(v if a == j else 5 for a in range(1, 4)) for j in range(1, 4) for v in (RB_XYZ[0] - 1, RB_XYZ[1] + 1)] + \
    [(RB_B[1], 65533, 65533, 65533)]


def rb_out_of_range(bad, seed=26):
    """(indices, row of `bad`): the accepted rows around the masked alias of `bad`, random rows, and `bad` at row 77."""
    rng = np.random.RandomState(seed)
    b, x, y, z = bad
    alias = np.array([b & 0xFFFF, x, y, z]) + np.array([0, -1, -1, -1])
    near = _block(alias[0], alias[1:])
    near = near[idx_ok(near)]
    rows = _unique_rows(rng, [near, _rb_size(200, seed)])
    rows = np.insert(rows, 77, np.asarray(bad, np.int32), axis=0)
    return rows.astype(np.int32), 77
