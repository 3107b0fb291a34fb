"""The edge cases tests/test_gpu_kernel_edges.py runs for the segment reductions (segment.cu), the row kernels
(voxelize.cu) and the instance-mask kernels (instances.cu), next to the launch constants those cases must reach.
tests/test_kernel_edges_coverage.py checks on the CPU that the table reaches every threshold below, so shrinking a case
fails there instead of quietly dropping the code path it was there for."""
import collections

import numpy as np

# launch constants of softgroup_b200/csrc
SEG_THREADS = 256  # segment.cu kSegThreads
SEG_CHUNK = 2048  # segment.cu kSegChunk: min / max partials are per 2048-row chunk
SEG_GRID = 132 * 4  # seg_minmax_kernel grid (SMs * 4, H100 SXM): more than SEG_GRID chunks take the grid-stride loop
MEAN_GRID = 65535  # seg_reduce_kernel / avg_pool_bp_kernel grid cap: more proposals take the grid-stride loop
SCAN_TILE = 512 * 8  # core.cu kScanTile: exclusive_scan_i32 has 2 levels above one tile, 3 above SCAN_TILE**2
PAN_THREADS = 1024  # instances.cu kPanThreads: one CTA walks the words of a mask


def pow2_cw(C):
    """Channel lanes of a segment CTA (segment.cu pow2_cw): the power of two >= min(C, 32)."""
    cw = 1
    while cw < C and cw < 32:
        cw <<= 1
    return cw


def rows_par(C):
    return SEG_THREADS // pow2_cw(C)


def bitmap_words(N):
    return (N + 1 + 31) // 32


def _offsets(lengths, start=0):
    return (start + np.concatenate([[0], np.cumsum(lengths)])).astype(np.int32)


def _lengths(n, total, seed, lo=1):
    """n lengths >= lo summing to total."""
    rng = np.random.RandomState(seed)
    cuts = np.sort(rng.choice(np.arange(1, total - n * lo + n), n - 1, replace=False))
    return np.diff(np.concatenate([[0], cuts, [total - n * lo + n]])) + lo - 1


# ---- segment min / max ----------------------------------------------------------------------------------------------
# kind: how test_gpu_kernel_edges fills the rows. 'specials': one- and two-row proposals of signed zeros, infinities, NaN,
# subnormals and +-FLT_MAX; 'negzero': an all -0.0 proposal and an all <= 0 proposal whose maximum -0.0 sits in one
# chunk; 'straddle': every proposal spans a chunk boundary, its extreme in one chunk and only {+0, -0, other sign} in
# the other, in both chunk orders; 'randn': negative-heavy normal values with signed zeros; 'lead': offsets[0] > 0, the
# rows below it hold values that would win.
MinMaxCase = collections.namedtuple('MinMaxCase', 'name C kind offsets')

_N_STRADDLE = 2000
_ALIGNED = np.array([0, 0, 0, 2048, 2048, 2048, 2048, 2100, 4096, 6144, 6144, 8192, 10240, 10240, 10240], np.int32)

MINMAX_CASES = [
    MinMaxCase('specials', 1, 'specials', _offsets([1] * 11 + [2] * 6)),
    MinMaxCase('specials_c3', 3, 'specials', _offsets([1] * 11 + [2] * 6)),
    MinMaxCase('negzero_3chunks', 3, 'negzero', _offsets([5000, 6200])),
    # proposal p >= 1 covers [1024 + 2048 (p-1), 1024 + 2048 p): half in chunk p-1, half in chunk p
    MinMaxCase('straddle', 1, 'straddle', _offsets([1024] + [SEG_CHUNK] * _N_STRADDLE)),
    MinMaxCase('straddle_c4', 4, 'straddle', _offsets([1024] + [SEG_CHUNK] * 600)),
    MinMaxCase('chunk_aligned_empty_runs', 5, 'randn', _ALIGNED),
    MinMaxCase('lead_rows', 3, 'lead', _offsets([900, 4000, 1, 3000], start=3000)),
    MinMaxCase('one_long_proposal', 3, 'randn', _offsets([2500000])),
    MinMaxCase('c2_proposals', 3, 'randn', _offsets(_lengths(40, 131761, seed=2, lo=50))),
] + [MinMaxCase('channels_%d' % C, C, 'randn', _offsets(_lengths(24, 30000, seed=C))) for C in
     (1, 2, 3, 4, 5, 8, 16, 31, 32, 33, 40, 64, 96)]

# ---- segment mean / global_avg_pool -----------------------------------------------------------------------------------
# data: 'relu' (non-negative, what global_avg_pool sees after the U-Net), 'offset' (1e4 + N(0,1): a large common offset),
# 'cancel' (+-1e3 alternating plus N(0, 1e-2): sums that cancel to far below sum |x|).
MeanCase = collections.namedtuple('MeanCase', 'name C data offsets')

_MANY = _offsets(np.random.RandomState(5).randint(0, 7, 70000))
_LONG = _offsets([200000, 1, 0, 37, 20000, 4095])

MEAN_CASES = [
    MeanCase('relu_long_c3', 3, 'relu', _LONG),
    MeanCase('relu_long_c32', 32, 'relu', _LONG),
    MeanCase('offset_long_c5', 5, 'offset', _LONG),
    MeanCase('cancel_long_c33', 33, 'cancel', _LONG),
    MeanCase('relu_many_c8', 8, 'relu', _MANY),
    MeanCase('cancel_many_c1', 1, 'cancel', _MANY),
] + [MeanCase('relu_c%d' % C, C, 'relu', _offsets(_lengths(12, 9000, seed=C + 100))) for C in (1, 2, 4, 16, 64, 96)]
ORACLE_REL_ROWS = 20000  # longest segment held to 1e-5 of the reference's own sequential float sum (see the test)

# ---- voxelize_fp / voxelize_bp: one voxel holding LONG_VOXEL points among ordinary voxels ------------------------------
LONG_VOXEL = 3000
VOXEL_CHANNELS = (3, 32, 35)

# ---- gather_rows: (name, N out rows, source rows, C, float offset of input, float offset of output) -------------------
GatherCase = collections.namedtuple('GatherCase', 'name N n_src C in_off out_off')
GATHER_CASES = [
    GatherCase('float4', 100003, 5000, 32, 0, 0),
    GatherCase('scalar_c3', 77777, 4000, 3, 0, 0),
    GatherCase('scalar_c5', 1, 7, 5, 0, 0),
    GatherCase('scalar_c33', 9999, 300, 33, 0, 0),
    GatherCase('misaligned_in', 50000, 1000, 32, 1, 0),
    GatherCase('misaligned_out', 50000, 1000, 16, 0, 1),
    GatherCase('full_size', 1500000, 1500000, 32, 0, 0),
]

# ---- instances: RLE of bitmaps ---------------------------------------------------------------------------------------
# Each case holds n_inst masks of N points; mask k has pattern PATTERNS[k % len] ('alternate' only for N <= 150000).
PATTERNS = ('empty', 'all', 'first', 'last', 'cross', 'random', 'alternate')
RleCase = collections.namedtuple('RleCase', 'name N n_inst')
RLE_CASES = [RleCase('n%d' % N, N, 7) for N in (1, 31, 32, 33, 63, 64, 65, 4096, 150000)] + [
    RleCase('one_tile_under', 4096, 31),  # 31 * 129 words = 3999
    RleCase('one_tile_exact', 4095, 32),  # 32 * 128 = 4096
    RleCase('one_tile_over', 4096, 32),  # 4128
    RleCase('three_level_scan', 1500000, 360),  # 360 * 46876 = 16,875,360 > 4096**2
]


def mask_of(pattern, N, seed):
    """Dense bool mask [N] of one pattern."""
    m = np.zeros(N, bool)
    if pattern == 'all':
        m[:] = True
    elif pattern == 'first':
        m[0] = True
    elif pattern == 'last':
        m[N - 1] = True
    elif pattern == 'alternate':
        m[seed % 2::2] = True
    elif pattern == 'cross':  # runs that start and end next to word boundaries, one ending at N - 1
        for a, b in ((30, 34), (63, 65), (95, 161), (N - 40, N)):
            m[max(a, 0):max(min(b, N), 0)] = True
    elif pattern == 'random':
        rng = np.random.RandomState(seed)
        k = min(64, N)
        edges = np.sort(rng.choice(N + 1, 2 * (k // 2), replace=False))
        for a, b in edges.reshape(-1, 2):
            m[a:b] = True
    return m


def rle_patterns(case):
    return [p for p in PATTERNS if p != 'alternate' or case.N <= 150000]


# ---- instances: count / scatter of mask scores ---------------------------------------------------------------------
# S entries (proposal, point); mask_scores [S, ms_stride], the first nI columns used; some scores exactly thr; keep
# leaves -1 holes in slot. layout: 'contiguous' (cluster order, proposals straddle warps), 'single' (one-entry
# proposals), 'interleaved' (ids shuffled within each warp: several match_any groups per warp).
InstCase = collections.namedtuple('InstCase', 'name S nP nI ms_stride N layout')
INST_CASES = [
    InstCase('contiguous_18', 10007, 173, 18, 18, 3001, 'contiguous'),
    InstCase('stride_over_nI', 20011, 311, 18, 24, 150000, 'contiguous'),
    InstCase('single_entries', 999, 999, 1, 1, 1025, 'single'),
    InstCase('interleaved', 8191, 97, 18, 20, 4096, 'interleaved'),
    InstCase('interleaved_1', 257, 9, 1, 3, 300, 'interleaved'),
]

# ---- instances: panoptic paste at the bench's size --------------------------------------------------------------------
PANOPTIC_N = 150000
PANOPTIC_INST = 720
