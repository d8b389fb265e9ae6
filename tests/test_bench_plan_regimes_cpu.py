"""CPU checks of the benchmark's inference plans (tests/bench_plan_cases.py): the configurations are the ones bench.py
times, together they reach every listed launch regime, and the mirrored size rules pick the plans the whole-network layer
lists of tests/test_gpu_model.py imply."""
import os
import sys

import pytest

import bench_plan_cases as bp
import test_gpu_train_step_kernels as ts

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


def _bench():
    sys.path.insert(0, ROOT)
    import bench
    return bench


def test_configurations_are_the_benchmarks():
    bench = _bench()
    cfg = {c['name']: c for c in bp.CONFIGS}
    for name in ('ssd300_b32_bf16x3', 'ssd300_b32_bf16'):
        c = cfg[name]
        assert (c['B'], c['n_classes'], c['mode'], c['pre']) == (bench.BATCH, bench.N_CLASSES, 'inference', {'divide_by_stddev': bench.STDDEV})
    assert bp.SC300 == bench.SC300
    assert {cfg[n]['prec'] for n in ('ssd300_b32_bf16x3', 'ssd300_b32_bf16')} == {'bf16x3', 'bf16'}
    assert (cfg['ssd512_b16_bf16x3']['B'], cfg['ssd512_b16_bf16x3']['n_classes'], cfg['ssd512_b16_bf16x3']['mode']) == (16, 80, 'inference_fast')
    assert (cfg['ssd7_b1_bf16x3']['B'], cfg['ssd7_b1_bf16x3']['n_classes']) == (1, 5)
    for c in bp.CONFIGS:                                   # the first and the last image of every batch are judged
        assert c['judged'][0] == 0 and c['judged'][-1] == c['B'] - 1


@pytest.mark.parametrize('cfg', bp.CONFIGS, ids=[c['name'] for c in bp.CONFIGS])
def test_configuration_reaches_its_regimes(cfg):
    got = bp.regimes(bp.build(cfg), cfg['B'])
    assert bp.EXPECTED[cfg['name']] <= got, (cfg['name'], sorted(got))


def test_configurations_reach_every_regime():
    reached = set()
    for cfg in bp.CONFIGS:
        reached |= bp.regimes(bp.build(cfg), cfg['B'])
    assert set(bp.REGIMES) <= reached, sorted(set(bp.REGIMES) - reached)
    assert set().union(*bp.EXPECTED.values()) == set(bp.REGIMES)


def _by_name(cfg):
    return {L['name']: L for L in bp.layers(bp.build(cfg), cfg['B'])}


def test_ssd300_plans_at_batch_32():
    """The layers of test_gpu_model's SSD300 lists: conv1_1 on the tensor cores with a gathered A tile, conv1_2 with the
    weights on the wgmma M side, the trunk on the implicit GEMM, the stride-2 extras on im2col, conv4_3_norm on l2norm8_kernel
    across both register halves, pool5 on the generic max-pool, and six fused heads at increasing prior offsets."""
    for cfg in bp.CONFIGS[:2]:
        L = _by_name(cfg)
        split = cfg['prec'] == 'bf16x3'
        assert L['conv1_1']['kernel'] == 'first_tc' and (L['conv1_1']['bn'], L['conv1_1']['kblocks']) == (64, 1)
        assert L['conv1_2']['kernel'] == 'gemm_swap' and L['conv1_2']['bm'] == 192
        for n in ('conv2_1', 'conv2_2', 'conv3_1', 'conv3_3', 'conv4_3', 'conv5_3', 'fc6', 'fc7', 'conv8_2', 'conv9_2'):
            assert L[n]['kernel'] == 'gemm', n
        assert L['conv6_2']['kernel'] == L['conv7_2']['kernel'] == 'im2col_gemm'
        assert L['conv6_2']['kblocks'] == 36 and L['conv4_3']['kblocks_per_tile'] == 72 and L['conv5_1']['kblocks_per_tile'] == 72
        assert [L['pool%d' % i]['kernel'] for i in range(1, 6)] == ['maxpool2x2'] * 4 + ['maxpool']
        assert L['conv4_3_norm']['kernel'] == 'l2norm8' and L['conv4_3_norm']['C'] == 512
        heads = [L[n] for n in L if n.endswith('_mbox')]
        assert len(heads) == 6 and all(h['head_fused'] for h in heads)
        assert [h['prior_off'] for h in heads] == [0, 5776, 7942, 8542, 8692, 8728]
        # conv5_x at 19 x 19 x 512: 105 m-tiles; bf16 keeps 256-wide tiles (two waves either way), bf16x3 takes 128
        assert L['conv5_1']['n_tiles_m'] == 105
        assert L['conv5_1']['bn'] == (128 if split else 256)


def test_ssd512_heads_are_unfused_with_81_classes():
    L = _by_name(bp.CONFIGS[2])
    heads = [L[n] for n in L if n.endswith('_mbox')]
    assert len(heads) == 7 and not any(h['head_fused'] for h in heads)
    assert {h['C'] for h in heads} == {4 * 85, 6 * 85}
    assert heads[-1]['prior_off'] + heads[-1]['H'] * heads[-1]['W'] * heads[-1]['n_boxes'] == 24564
    assert L['conv10_2']['k'] == 4 and L['conv10_2']['kernel'] == 'gemm'


def test_ssd7_plan_folds_batchnorm_into_every_epilogue():
    L = _by_name(bp.CONFIGS[3])
    assert L['conv1']['kernel'] == 'first_tc' and L['conv1']['kblocks'] == 2 and L['conv1']['bn'] == 64
    for i in range(1, 8):
        assert L['conv%d' % i]['bn_layer'] == 'bn%d' % i and L['conv%d' % i]['act'] == 'elu'
    assert all(L['conv%d' % i]['kernel'] == 'gemm' for i in range(2, 8))
    assert all(L['pool%d' % i]['kernel'] == 'maxpool2x2' for i in range(1, 7))
    heads = [L['head%d' % i] for i in (4, 5, 6, 7)]
    assert all(h['head_fused'] for h in heads) and heads[0]['prior_off'] == 0 and heads[1]['prior_off'] > 0


def test_mirrors_agree_with_the_per_launch_tables():
    """The rules here and the per-launch suites' own mirrors pick the same kernels."""
    for C in (20, 32, 264, 512, 520):
        assert bp.l2norm_kernel_of(C) == ts.l2norm_kernel_of(C, -(-C // 8) * 8)
    for c in ts.POOL_CASES:
        assert bp.pool_kernel_of(c['H'], c['W'], c['k'], c['stride'], c['pads']) == c['kernel']
    # the wave rule: few m-tiles leave a 256-wide last wave mostly empty, 105 m-tiles of 512 channels do not
    assert bp.gemm_bn(512, False, 105) == 256 and bp.gemm_bn(512, False, 70) == 128 and bp.gemm_bn(512, True, 105) == 128
    assert bp.gemm_bn(264, False, 3) == 256 and bp.gemm_bn(150, True, 3) == 160
    assert bp.valid_tiles(1, 3, 130, 2, 128, 128) == 3 and bp.valid_tiles(2, 12, 11, 10, 10, 128) == 2
