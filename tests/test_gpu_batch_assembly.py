"""Device-side batch assembly (ssdk_assemble_batch) against label arrays produced by the REAL reference's CropPad / Flip /
Resize / BoxFilter in the order of the original SSD augmentation chain (tests/golden/make_batch_golden.py), and the
assembled batch fed straight into the encoder without a host round trip."""
import json
import os

import numpy as np
import pytest

import assembly_cases as ac

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'ref_batch_golden.npz'))
META = json.load(open(os.path.join(HERE, 'golden', 'ref_batch_golden.json')))


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


def _ops(lst):
    from ssd_keras_b200.data_generator import batch_assembly as ba
    out = []
    for o in lst:
        if o[0] == 'crop_pad':
            out.append(ba.crop_pad(o[1], o[2], o[3], o[4], center_point_filter=o[5], clip_boxes=o[6]))
        elif o[0] == 'flip':
            out.append(ba.flip(o[1], o[2]))
        elif o[0] == 'resize':
            out.append(ba.resize(o[1], o[2], o[3], o[4], drop_degenerate=o[5]))
        else:
            out.append(ba.box_filter(check_degenerate=o[1], min_area=o[2]))
    return out


def test_box_ops_match_reference_chain():
    from ssd_keras_b200.data_generator.batch_assembly import assemble_batch_device
    B = META['n']
    labels = [G['in%d' % b] for b in range(B)]
    gt, offs, stats, total, max_g = assemble_batch_device(labels, [_ops(o) for o in META['ops']])
    gt, offs, stats = gt.cpu().numpy(), offs.cpu().numpy(), stats.cpu().numpy()
    assert offs[0] == 0 and total == sum(l.shape[0] for l in labels) and max_g == max(l.shape[0] for l in labels)
    for b in range(B):
        ref = G['out%d' % b]
        ac.assert_f32_bits(gt[offs[b]:offs[b + 1]], ref, 'image %d' % b)                  # same boxes, same order, same bits
    assert stats[0] == offs[-1] == sum(G['out%d' % b].shape[0] for b in range(B))
    assert stats[1] == max(G['out%d' % b].shape[0] for b in range(B))
    # pack only (no operations): the identity
    gt2, offs2, _, _, _ = assemble_batch_device(labels)
    ac.assert_f32_bits(gt2.cpu().numpy()[:total], np.concatenate(labels), 'pack only')
    np.testing.assert_array_equal(offs2.cpu().numpy(), np.cumsum([0] + [l.shape[0] for l in labels]))


def test_assembled_batch_feeds_the_encoder(configs):
    """generate() -> label_encoder(batch_y): boxes transformed, filtered and packed on the device go to the encoder through
    device-resident offsets; the result equals encoding the reference-transformed labels."""
    from ssd_keras_b200.data_generator.batch_assembly import encode_batch_device
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    B = META['n']
    labels = [G['in%d' % b] for b in range(B)]
    enc = SSDInputEncoder(**configs['ssd300'])
    y = encode_batch_device(enc, labels, [_ops(o) for o in META['ops']]).cpu().numpy()
    y_ref = enc([G['out%d' % b] for b in range(B)])
    np.testing.assert_array_equal(y, y_ref.astype(np.float32))
