"""One table of sparse-convolution problems for the tensor-core kernel (softgroup_b200/csrc/spconv_tc.cu), and the launch
each of them gets.

BENCH_CASES are the convolutions of the 150k-point `c2_scannet` bench scan (seed 0, scannet config 32 x 7) with its real
level sizes; SYNTHETIC_CASES reach the tile configurations the bench does not (NT = 16 / 48 / 80 / 112 / 128 in the
one-CTA-per-item form, split-K with a ragged last column part, split-K sizes 2 and 4-7, odd Cout, a last 32-channel slice
of 17-31 channels, Cin up to 512, empty tiles). tests/test_spconv_coverage.py checks on the CPU that the table reaches
every configuration; tests/test_gpu_spconv_configs.py runs every case on the GPU against the float64 oracle."""
from collections import namedtuple

# rows per U-Net level of the bench scan (voxelization_idx(coords, 1, 4), then one k2 s2 rulebook per level)
BENCH_ROWS = (137100, 101434, 42391, 10345, 1933, 332, 52)
BENCH_CHANNELS = tuple(32 * (i + 1) for i in range(len(BENCH_ROWS)))
BENCH_SEED, BENCH_POINTS = 0, 150000
H100_SMS = 132  # H100 SXM5; the launch uses the device's own count

# kind: 'subm' (27-offset rulebook of the level), 'down' (k2 s2: level -> level + 1), 'inv' (its inverse: level + 1 ->
# level), 'ident' (1x1, no map), 'rand' (synthetic K-offset rulebook of random rows, Min input rows)
Case = namedtuple('Case', 'name kind level K Mout Min Cin Cout')


def _bench_cases():
    M, C = BENCH_ROWS, BENCH_CHANNELS
    cases = [Case('input_conv', 'subm', 0, 27, M[0], M[0], 6, C[0])]
    for i in range(len(M)):
        cases.append(Case('subm%d' % i, 'subm', i, 27, M[i], M[i], C[i], C[i]))
        if i + 1 == len(M):
            break
        cases += [
            Case('down%d' % i, 'down', i, 8, M[i + 1], M[i], C[i], C[i + 1]),
            Case('inv%d' % i, 'inv', i, 8, M[i], M[i + 1], C[i + 1], C[i]),
            Case('tail_subm%d' % i, 'subm', i, 27, M[i], M[i], 2 * C[i], C[i]),  # first block after the concat
            Case('tail_1x1_%d' % i, 'ident', i, 1, M[i], M[i], 2 * C[i], C[i]),  # its 1x1 identity branch
        ]
    return cases


BENCH_CASES = _bench_cases()

SYNTHETIC_CASES = [
    Case('nt16_odd', 'rand', None, 27, 3000, 2500, 40, 13),           # Cout <= 16: NT = 16 in both forms
    Case('nt16_many_tiles', 'rand', None, 8, 20000, 9000, 24, 16),   # NT = 16, last slice of 24 channels
    Case('nt48', 'rand', None, 27, 20000, 18000, 48, 48),            # NT = 48 in both forms
    Case('nt80', 'rand', None, 8, 9000, 30000, 96, 160),             # NT = 80 x 2 in both forms
    Case('nt112', 'rand', None, 27, 9000, 9000, 200, 224),           # NT = 112 x 2 in both forms
    Case('nt128_x2', 'ident', None, 1, 9000, 9000, 130, 250),        # NT = 128 x 2, 1x1 identity
    Case('nt96_ragged', 'rand', None, 8, 5000, 5000, 120, 176),      # persistent 96 + 80, last slice 24 channels
    Case('splitk8_ragged', 'rand', None, 27, 100, 400, 300, 199),    # 32 x 7 (last part 16 wide) with S = 8, odd Cout
    Case('splitk2_ident', 'ident', None, 1, 300, 300, 256, 64),      # S = 2
    Case('splitk6', 'rand', None, 27, 1280, 1500, 64, 128),          # 10 tiles x 4 parts: S = 2 sms / 40
    Case('splitk_cin512', 'rand', None, 8, 200, 700, 512, 256),      # Cin = 512 (16 slices), Cout = 256
    Case('splitk3_cin448', 'ident', None, 1, 520, 600, 448, 112),    # S = 3 from K * nkc / 4, last slice 0 mod 32
]

CASES = BENCH_CASES + SYNTHETIC_CASES


def div_up(a, b):
    return -(-a // b)


def persistent_nt(N):
    """Columns per work item of the persistent launch -- `persistent_nt` in softgroup_b200/csrc/spconv_tc.cu."""
    return N if N <= 128 else (div_up(N, div_up(N, 128)) + 15) // 16 * 16


def launch(case, form, sms, L):
    """The launch of `case` in form 0 (one CTA per work item) or 1 (persistent), through the library's pure plan
    functions: dict(NT, parts, last (columns of the last part), S, tiles, items, nkc, ks_last)."""
    import ctypes
    N = (case.Cout + 15) // 16 * 16
    tiles = div_up(case.Mout, 128)
    if form == 1:
        NT, S = persistent_nt(N), 1
    else:
        out = (ctypes.c_int * 6)()
        assert L.sgb_spconv_tc_plan(case.K, case.Mout, case.Cin, case.Cout, int(case.kind != 'ident'), sms, out) == 0
        NT, S = out[0], out[2]
        assert out[1] == div_up(N, NT) and out[5] == tiles
    parts = div_up(N, NT)
    nkc = div_up(case.Cin, 32)
    return dict(NT=NT, parts=parts, last=N - (parts - 1) * NT, S=S, tiles=tiles, items=tiles * parts, nkc=nkc,
                ks_last=(case.Cin - (nkc - 1) * 32 + 15) >> 4)
