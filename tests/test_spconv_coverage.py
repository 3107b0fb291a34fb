"""CPU: the case table of tests/spconv_cases.py reaches every tile configuration of the tensor-core convolution kernel
(spconv_tc.cu), mapped to launches through the library's pure plan functions (sgb_spconv_tc_plan,
sgb_spconv_kernel_choice); no GPU compute. tests/test_gpu_spconv_configs.py runs each case under both launch forms, so a
configuration reached here is a configuration compared with the float64 oracle there."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import spconv_cases as sc  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402


def _sms():
    """132 (H100 SXM5) without a GPU; the device's own count with one, as the launch uses it."""
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:
        pass
    return sc.H100_SMS


def test_persistent_nt_matches_the_library():
    """The Python restatement of persistent_nt agrees with what the library reports for N <= 128, where the
    one-CTA-per-item plan with many row tiles also takes all N columns."""
    L = _lib.lib()
    for N in range(16, 129, 16):
        a = sc.launch(sc.Case('x', 'rand', None, 27, 1 << 20, 1 << 20, 32, N), 0, 132, L)
        assert a['NT'] == N == sc.persistent_nt(N)
    assert [sc.persistent_nt(N) for N in range(144, 257, 16)] == [80, 80, 96, 96, 112, 112, 128, 128]


def test_case_table_is_well_formed():
    names = [c.name for c in sc.CASES]
    assert len(set(names)) == len(names)
    for c in sc.CASES:
        assert 1 <= c.Cin <= 512 and 1 <= c.Cout <= 256 and c.K in (1, 8, 27)
        assert c.kind in ('subm', 'down', 'inv', 'ident', 'rand')
        assert c.kind != 'ident' or (c.K == 1 and c.Min >= c.Mout)
        assert (c.level is None) == (c in sc.SYNTHETIC_CASES) and (c.kind == 'rand') <= (c.level is None)
    # the bench table: every convolution kind of every level at the scan's row counts
    M, C = sc.BENCH_ROWS, sc.BENCH_CHANNELS
    by = {c.name: c for c in sc.BENCH_CASES}
    assert by['down3'][3:] == (8, M[4], M[3], 128, 160) and by['tail_1x1_5'][3:] == (1, M[5], M[5], 384, 192)
    assert by['subm6'][3:] == (27, M[6], M[6], 224, 224) and len(sc.BENCH_CASES) == 1 + 7 + 4 * 6


@pytest.mark.parametrize('sms', sorted({sc.H100_SMS, _sms()}))
def test_case_table_reaches_every_tile_configuration(sms):
    L = _lib.lib()
    seen = {'nt0': set(), 'nt1': set(), 'S': set(), 'K': set(), 'ks_last': set(), 'last_slice': set()}
    split_ragged = cin_big = odd_cout = persistent_overfull = False
    for c in sc.CASES:
        a, b = sc.launch(c, 0, sms, L), sc.launch(c, 1, sms, L)
        seen['nt0'].add(a['NT'])
        seen['nt1'].add(b['NT'])
        seen['S'].add(a['S'])
        seen['K'].add(c.K)
        seen['ks_last'].add(a['ks_last'])
        seen['last_slice'].add('1-16' if 1 <= c.Cin % 32 <= 16 else ('17-31' if c.Cin % 32 > 16 else '32'))
        split_ragged |= a['S'] > 1 and a['parts'] > 1 and a['last'] < a['NT']
        cin_big |= c.Cin > 256
        odd_cout |= c.Cout % 2 == 1
        # a persistent CTA holds at most 2 per SM (launch bounds + shared memory): more items than that many CTAs
        persistent_overfull |= b['items'] > 2 * sms
        assert L.sgb_spconv_kernel_choice(c.K, c.Mout, c.Cin, c.Cout, sms) in (0, 1)
    every_nt = set(range(16, 129, 16))
    assert seen['nt0'] == every_nt, 'one CTA per item: NT %s' % sorted(seen['nt0'])
    assert seen['nt1'] == every_nt, 'persistent: NT %s' % sorted(seen['nt1'])
    assert {1, 2, 3, 8} <= seen['S'] and seen['S'] & {4, 5, 6, 7}, 'split-K %s' % sorted(seen['S'])
    assert seen['K'] == {1, 8, 27}
    assert seen['ks_last'] == {1, 2} and {'1-16', '17-31'} <= seen['last_slice']
    assert split_ragged, 'split-K with several column parts, the last narrower than NT'
    assert cin_big and odd_cout and persistent_overfull


def test_bench_cases_take_the_documented_launches():
    """The launches the 150k-point bench runs per level, on an H100 SXM5 (132 SMs): persistent with all columns up to
    level 3, persistent 80 x 2 at Cout 160, one CTA per item with split-K clusters at levels 5-6."""
    L = _lib.lib()
    by = {c.name: c for c in sc.BENCH_CASES}
    choice = {n: L.sgb_spconv_kernel_choice(c.K, c.Mout, c.Cin, c.Cout, sc.H100_SMS) for n, c in by.items()}
    for n in ('subm0', 'tail_1x1_0', 'down2', 'subm3', 'inv3', 'tail_subm3', 'down3', 'subm4', 'inv4', 'tail_1x1_4'):
        assert choice[n] == 1, n
    for n in ('down3', 'subm4', 'inv4', 'tail_subm4', 'tail_1x1_4'):
        b = sc.launch(by[n], 1, sc.H100_SMS, L)
        assert (b['NT'], b['parts']) == (80, 2), n
    for n in ('down4', 'subm5', 'inv5', 'tail_subm5', 'down5', 'subm6'):
        a = sc.launch(by[n], 0, sc.H100_SMS, L)
        assert choice[n] == 0 and a['NT'] == 32 and a['S'] == 8, n
    a = sc.launch(by['tail_1x1_5'], 0, sc.H100_SMS, L)
    assert choice['tail_1x1_5'] == 0 and (a['NT'], a['parts'], a['S']) == (32, 6, 3)
