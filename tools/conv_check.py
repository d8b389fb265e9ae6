#!/usr/bin/env python
"""Debug harness for the wgmma conv path: small graphs, every layer compared with torch-CPU float32.
Each case runs in its own process so that a device trap in one case cannot poison the others.
Usage (GPU box):  python tools/conv_check.py            # all cases
                  python tools/conv_check.py --case 3   # one case, in-process
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)

CASES = [
    # name, image HxW, batch, layers [(name, cout, k, stride, dilation, pad, act)], precision
    ('im2col_3to64', 16, 1, [('c1', 64, 3, 1, 1, 1, 1)], 'bf16x3'),
    ('virt_64to64', 16, 2, [('c1', 64, 3, 1, 1, 1, 1), ('c2', 64, 3, 1, 1, 1, 1)], 'bf16x3'),
    ('virt_bn128_256', 20, 2, [('c1', 64, 3, 1, 1, 1, 1), ('c2', 128, 3, 1, 1, 1, 1), ('c3', 256, 3, 1, 1, 1, 1)], 'bf16x3'),
    ('ntiles2_1x1_dil', 19, 2, [('c1', 64, 3, 1, 1, 1, 1), ('c2', 512, 3, 1, 1, 1, 1), ('c3', 256, 1, 1, 1, 0, 1),
                                ('c4', 128, 3, 1, 6, 6, 1)], 'bf16x3'),
    ('stride2_valid_4x4', 21, 2, [('c1', 64, 3, 1, 1, 1, 1), ('c2', 128, 3, 2, 1, 1, 1), ('c3', 64, 3, 1, 1, 0, 1),
                                  ('c4', 64, 4, 1, 1, 1, 0)], 'bf16x3'),
    ('odd_channels_elu', 24, 2, [('c1', 32, 5, 1, 1, 2, 2), ('c2', 48, 3, 1, 1, 1, 2), ('c3', 64, 3, 1, 1, 1, 2)], 'bf16x3'),
    ('single_pass_bf16', 16, 2, [('c1', 64, 3, 1, 1, 1, 1), ('c2', 64, 3, 1, 1, 1, 1)], 'bf16'),
    ('big_m_persistent', 150, 4, [('c1', 64, 3, 1, 1, 1, 1), ('c2', 64, 3, 1, 1, 1, 1)], 'bf16x3'),
]


def run_case(i):
    import torch
    import torch.nn.functional as Fn
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.models._graph import SSDModel, Spec, same_pad
    name, hw, B, layers, prec = CASES[i]
    specs = [Spec('input', _ffi.OP_INPUT, params={'mean': [123, 117, 104], 'stddev': None, 'swap': [2, 1, 0]})]
    prev = 'input'
    for (n, cout, k, s, d, p, act) in layers:
        specs.append(Spec(n, _ffi.OP_CONV, prev, cout=cout, k=(k, k), stride=s, dilation=d, pad=(p, p, p, p), act=act))
        prev = n
    specs.append(Spec('head', _ffi.OP_HEAD, prev, k=(3, 3), pad=same_pad(3), n_boxes=3, params={'conf_name': 'hc', 'loc_name': 'hl'}))
    n_cls = 5
    anchor_cfg = dict(scales=[0.2, 0.4], aspect_ratios_per_layer=[[1.0, 2.0]], two_boxes_for_ar1=True, steps=None, offsets=None,
                      clip_boxes=False, coords='centroids', normalize_coords=True)
    m = SSDModel(specs, hw, hw, 3, n_cls, anchor_cfg, [0.1, 0.1, 0.2, 0.2], 'training', {}, precision=prec, seed=3)
    rng = np.random.default_rng(7)
    w = m.get_weights()
    for k_ in w:
        if k_.endswith('/bias'):
            w[k_] = (rng.standard_normal(w[k_].shape) * 0.1).astype(np.float32)
    m.set_weights(w)
    x = rng.integers(0, 256, size=(B, hw, hw, 3)).astype(np.float32)
    y = m.predict(x)
    torch.cuda.synchronize()
    # torch-CPU float32 reference
    t = torch.from_numpy(x) - torch.tensor([123., 117., 104.])
    t = t[..., [2, 1, 0]].permute(0, 3, 1, 2).contiguous()
    worst = 0.0
    for (n, cout, k, s, d, p, act) in layers:
        kw = torch.from_numpy(np.ascontiguousarray(np.transpose(w[n + '/kernel'], (3, 2, 0, 1))))
        t = Fn.conv2d(t, kw, torch.from_numpy(w[n + '/bias']), stride=s, padding=p, dilation=d)
        t = torch.relu(t) if act == 1 else (Fn.elu(t) if act == 2 else t)
        got = m.read_layer(n, B)
        ref = t.permute(0, 2, 3, 1).numpy()
        err = np.abs(got - ref).max(); scale = np.abs(ref).max() + 1e-30
        nbad = int((np.abs(got - ref) > 1e-3 * scale + 1e-3).sum())
        print('  case %d %-18s layer %-4s shape %-18s max|err| %.3e  max|ref| %.3e  rel %.2e  bad %d/%d'
              % (i, name, n, str(got.shape), err, scale, err / scale, nbad, got.size), flush=True)
        worst = max(worst, err / scale)
        if nbad and nbad < got.size:
            idx = np.argwhere(np.abs(got - ref) > 1e-3 * scale + 1e-3)
            print('    first bad (n,y,x,c):', idx[:6].tolist(), 'got', got[tuple(idx[0])], 'ref', ref[tuple(idx[0])], flush=True)
    hc = Fn.conv2d(t, torch.from_numpy(np.ascontiguousarray(np.transpose(w['hc/kernel'], (3, 2, 0, 1)))), torch.from_numpy(w['hc/bias']), padding=1)
    hl = Fn.conv2d(t, torch.from_numpy(np.ascontiguousarray(np.transpose(w['hl/kernel'], (3, 2, 0, 1)))), torch.from_numpy(w['hl/bias']), padding=1)
    conf = torch.softmax(hc.permute(0, 2, 3, 1).reshape(B, -1, n_cls), -1).numpy()
    loc = hl.permute(0, 2, 3, 1).reshape(B, -1, 4).numpy()
    e1 = np.abs(y[:, :, :n_cls] - conf).max(); e2 = np.abs(y[:, :, n_cls:n_cls + 4] - loc).max() / (np.abs(loc).max() + 1e-30)
    e3 = np.abs(y[:, :, n_cls + 4:n_cls + 8] - m.anchors_f32[None]).max()
    print('  case %d %-18s head: softmax err %.3e  loc rel err %.3e  anchor err %.1e' % (i, name, e1, e2, e3), flush=True)
    tol = 3e-2 if prec == 'bf16' else 2e-4
    ptol = tol * max(1.0, float(hc.abs().max()))          # probabilities move by up to |d logit|
    ok = worst < tol and e1 < ptol and e2 < tol and e3 == 0
    print('CASE %d %s: %s' % (i, name, 'OK' if ok else 'FAIL'), flush=True)
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--case', type=int, default=-1)
    args = ap.parse_args()
    if args.case >= 0:
        sys.exit(run_case(args.case))
    import __graft_entry__
    __graft_entry__.build()
    bad = 0
    for i in range(len(CASES)):
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), '--case', str(i)], capture_output=True, text=True, timeout=300)
            out = (r.stdout + r.stderr)
            print(out[-3000:], flush=True)
            bad += (r.returncode != 0)
        except subprocess.TimeoutExpired:
            print('CASE %d TIMEOUT' % i, flush=True)
            bad += 1
    print('conv_check: %d/%d cases failed' % (bad, len(CASES)))
    sys.exit(1 if bad else 0)


if __name__ == '__main__':
    main()
