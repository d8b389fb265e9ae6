"""CPU-side checks: the C-ABI library builds/loads, exports every declared symbol, host-only entry points
(anchors) match the golden vectors, and the Python mirror validates arguments like the reference."""
import ctypes
import hashlib
import os
import re

import numpy as np
import pytest

import __graft_entry__ as entry

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


@pytest.fixture(scope='module')
def lib():
    entry.build()
    from ssd_keras_b200 import _ffi
    return _ffi.lib()


HEADER_KINDS = {'int': 'i32', 'long long': 'i64', 'int64_t': 'i64', 'float': 'f32', 'double': 'f64', 'void': 'void'}


def _header():
    """include/ssdk.h without its comments."""
    src = open(os.path.join(ROOT, 'include', 'ssdk.h')).read()
    return re.sub(r'//[^\n]*', '', re.sub(r'/\*.*?\*/', ' ', src, flags=re.S))


def _declarators(decl):
    """'const int* a, b[4]' -> [(name, kind, array length or None)]; a pointer is 'ptr', a scalar its HEADER_KINDS kind."""
    first, *more = re.sub(r'\bconst\b', ' ', decl).split(',')
    base, d0 = re.fullmatch(r'\s*([\w\s]*?\w)((?:\s|\*)*\w*\s*(?:\[\d+\])?)\s*', first).groups()
    out = []
    for d in [d0] + more:
        stars, name, n = re.fullmatch(r'\s*(\**)\s*(\w*)\s*(?:\[(\d+)\])?\s*', d).groups()
        out.append((name, 'ptr' if stars else HEADER_KINDS[base], int(n) if n else None))
    return out


def _ctypes_kind(t):
    if t is None:
        return 'void'
    if issubclass(t, (ctypes._Pointer, ctypes.c_void_p, ctypes.c_char_p)):
        return 'ptr'
    return {'f': 'f32', 'd': 'f64'}.get(t._type_, 'i%d' % (8 * ctypes.sizeof(t)))


def test_binding_table_matches_the_header(lib):
    """_ffi.SIGNATURES declares exactly the functions of ssdk.h, each exported, with the header's arity and the kind (pointer,
    32- / 64-bit int, float, double) of every argument and return value; each ctypes Structure of _ffi (named after its C
    struct: BoxOp mirrors ssdk_box_op) has the header's fields in order, with the same kinds and array lengths."""
    from ssd_keras_b200 import _ffi
    header = _header()
    decls = {name: (ret, params) for ret, name, params in
             re.findall(r'((?:const\s+)?\w+\s*\**)\s*\b(ssdk_\w+)\s*\(([^()]*)\)\s*;', header)}
    assert sorted(decls) == sorted(_ffi.SIGNATURES)
    for name, (ret, params) in decls.items():
        assert hasattr(lib, name), 'libssdk.so does not export ' + name
        restype, argtypes = _ffi.SIGNATURES[name]
        want = [k for p in params.split(',') if p.strip() != 'void' for _, k, _ in _declarators(p)]
        assert (_declarators(ret + ' r')[0][1], want) == (_ctypes_kind(restype), [_ctypes_kind(t) for t in argtypes]), name
    assert lib.ssdk_version() == 100
    structs = {name: body for body, name in re.findall(r'typedef\s+struct\s*\w*\s*\{([^{}]*)\}\s*(\w+)\s*;', header)}
    mirrors = [c for c in vars(_ffi).values() if isinstance(c, type) and issubclass(c, ctypes.Structure)]
    assert mirrors
    for cls in mirrors:
        c_name = 'ssdk_' + re.sub(r'(?<!^)([A-Z])', r'_\1', cls.__name__).lower()
        assert c_name in structs, (cls.__name__, c_name)
        want = [f for decl in structs[c_name].split(';') if decl.strip() for f in _declarators(decl)]
        have = [(n, _ctypes_kind(t._type_ if issubclass(t, ctypes.Array) else t), t._length_ if issubclass(t, ctypes.Array) else None)
                for n, t in cls._fields_]
        assert have == want, cls.__name__


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    h = ctypes.c_void_p()
    rc = lib.ssdk_ctx_create(0, ctypes.byref(h))
    assert rc == -2 and b'no CPU fallback' in lib.ssdk_last_error()
    from ssd_keras_b200 import _ffi
    with pytest.raises(_ffi.SSDKError):
        _ffi.context()


def sha16(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


@pytest.mark.parametrize('name', ['ssd300', 'ssd512', 'ssd7', 'micro', 'tiny', 'tiny_clip_abs'])
def test_anchors_match_reference(lib, golden, configs, name):
    """ssdk_anchors_generate (host float64) against anchors produced by the real reference encoder."""
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    arr, meta = golden
    enc = SSDInputEncoder(**configs[name])
    m = meta['anchors/' + name]
    assert enc.anchors.shape == (m['P'], 4)
    assert sha16(enc.anchors_f32) == m['sha_f32']
    assert enc.anchors[0].tolist() == m['first'] and enc.anchors[-1].tolist() == m['last']
    assert abs(enc.anchors.sum() - m['sum']) < 1e-9 * abs(m['sum'])
    assert enc.n_boxes == m['n_boxes']
    if name.startswith('tiny'):
        np.testing.assert_array_equal(enc.anchors, arr['anchors/' + name])      # bit-exact float64
    assert len(enc.boxes_list) == len(configs[name]['predictor_sizes'])
    # for coords='minmax'/'corners' too
    for co in ('corners', 'minmax'):
        from oracle.encoder import OracleEncoder
        c = dict(configs[name]); c['coords'] = co
        np.testing.assert_array_equal(SSDInputEncoder(**c).anchors, OracleEncoder(**c).anchors)


def test_encoder_argument_validation(lib, configs):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    base = dict(configs['tiny'])
    for bad in (dict(scales=[0.1, 0.2]), dict(scales=None, min_scale=None), dict(variances=[0.1, 0.1]),
                dict(variances=[0.1, 0.1, 0.0, 0.2]), dict(coords='polar'), dict(steps=[8]), dict(offsets=[0.5]),
                dict(aspect_ratios_per_layer=[[1.0]]), dict(aspect_ratios_global=[-1.0])):
        c = dict(base); c.update(bad)
        with pytest.raises(ValueError):
            SSDInputEncoder(**c)


def test_model_builders_shapes_and_validation(lib):
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    from ssd_keras_b200.models.keras_ssd512 import ssd_512
    from ssd_keras_b200.models.keras_ssd7 import build_model, ssd_7
    m, ps = ssd_300((300, 300, 3), 20, scales=[0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05], return_predictor_sizes=True)
    assert ps.tolist() == [[38, 38], [19, 19], [10, 10], [5, 5], [3, 3], [1, 1]] and m.n_boxes_total == 8732
    assert m.get_layer('conv4_3_norm_mbox_conf').output_shape == (None, 38, 38, 84)
    assert m.get_layer('fc7_mbox_loc').output_shape[1:3] == (19, 19)
    assert sum(int(np.prod(v.shape)) for k, v in m.get_weights().items()) == 26285486      # SURVEY K13
    m, ps = ssd_512((512, 512, 3), 80, scales=[0.04, 0.1, 0.26, 0.42, 0.58, 0.74, 0.9, 1.06], return_predictor_sizes=True)
    assert ps[:, 0].tolist() == [64, 32, 16, 8, 4, 2, 1] and m.n_boxes_total == 24564
    m, ps = build_model((300, 300, 3), 5, scales=[0.08, 0.16, 0.32, 0.64, 0.96], return_predictor_sizes=True)
    assert ps[:, 0].tolist() == [37, 18, 9, 4] and m.n_boxes_total == 7160 and ssd_7 is build_model
    with pytest.raises(ValueError):
        ssd_300((300, 300, 3), 20, mode='bogus', scales=[0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05])
    with pytest.raises(ValueError):
        ssd_300((300, 300, 3), 20, scales=[0.1, 0.2])
    with pytest.raises(ValueError):
        ssd_300((300, 300, 3), 20)                       # neither scales nor min/max
    with pytest.raises(ValueError):
        ssd_300((300, 300, 3), 20, min_scale=0.1, max_scale=0.9, steps=[8, 16])


def test_decode_layer_argument_validation(lib):
    from ssd_keras_b200.keras_layers.keras_layer_DecodeDetections import DecodeDetections
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_detections
    with pytest.raises(ValueError):
        DecodeDetections(coords='corners', img_height=300, img_width=300)
    with pytest.raises(ValueError):
        DecodeDetections(normalize_coords=True)
    with pytest.raises(ValueError):
        decode_detections(np.zeros((1, 4, 16), np.float32))   # normalize_coords without image size


def test_product_never_imports_oracle():
    """The shipped package must not reference the oracle (it is test infrastructure)."""
    pkg = os.path.join(ROOT, 'ssd_keras_b200')
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh')):
                src = open(os.path.join(dp, f)).read()
                assert 'import oracle' not in src and 'from oracle' not in src, f
