"""The case tables and conv_swap_kernel (SSDK_PLAN_GEMM_SWAP): the swapped-operand cases reach the variant in both precisions,
with every shape the kernel has to handle, and no case of the other tables does -- those keep pinning the 128-pixel kernels.
The plan builder's rule is mirrored in tests/swap_cases.py."""
import conv_cases as cc
import swap_cases as sc


def _pixels(c):
    ph = c['pads'][0] + c['pads'][2]
    pw = c['pads'][1] + c['pads'][3]
    eff = c['dil'] * (c['k'] - 1) + 1
    return c['B'] * ((c['H'] + ph - eff) // c['stride'] + 1) * ((c['W'] + pw - eff) // c['stride'] + 1)


def test_swap_case_table_reaches_the_variant():
    cases = sc.SWAP_CASES
    for c in cases:
        assert c['expect']['kernel'] == 'gemm_swap' and c['expect']['bm'] == 192, c['name']
        assert sc.selects_swap(c['cin'], c['cout'], c['stride'], _pixels(c)), c['name']
    assert {c['expect']['split'] for c in cases} == {0, 1}
    for split in (0, 1):
        mine = [c for c in cases if c['expect']['split'] == split]
        assert any(c['cout'] == 64 for c in mine) and any(c['cout'] < 64 for c in mine)           # full and partial tile
        assert any(c['cin'] == 128 for c in mine)                                                 # two k-blocks
        assert any(c['B'] > 1 and (c['H'] + 2) * (c['W'] + 1) % 192 for c in mine)                # an image ends inside a tile
        assert {c['env'].get('SSDK_SHARED_BORDER', '1') for c in mine} == {'0', '1'}
        assert {c['act'] for c in mine} == {'relu', None, 'elu'}
    assert any(c['bn'] for c in cases) and any(not c['bias'] for c in cases)


def test_no_other_case_table_reaches_the_variant():
    for c in cc.FORWARD_CASES:
        assert c['expect']['kernel'] != 'gemm_swap'
        assert not sc.selects_swap(c['cin'], c['cout'], c['stride'], _pixels(c)), c['name']
    for c in cc.HEAD_CASES:
        assert c['expect']['kernel'] != 'gemm_swap'
        assert not sc.selects_swap(c['cin'], c['nb'] * (c['C'] + 4), 1, c['B'] * c['H'] * c['W'], head=True), c['name']


def test_the_rule_takes_conv1_2_of_ssd300_and_ssd512():
    assert sc.selects_swap(64, 64, 1, 32 * 300 * 300)
    assert sc.selects_swap(64, 64, 1, 8 * 512 * 512)
    assert not sc.selects_swap(64, 128, 1, 32 * 150 * 150)               # conv2_1: 128 output channels
    assert not sc.selects_swap(32, 64, 1, 32 * 300 * 300)                # too few input channels
    assert not sc.selects_swap(64, 64, 2, 32 * 300 * 300)                # strided: im2col
    assert not sc.selects_swap(64, 64, 1, 2 * 132 * 192 - 1)             # fewer than two 192-pixel tiles per SM
