#!/usr/bin/env python
"""Per-layer timing of the conv_wgmma_kernel launches of the benchmark's model: SSD300, batch 32, mode='inference',
divide_by_stddev, bf16x3 (or bf16 with `fast`).  CUDA events around every launch, on one stream (the instrumented forward does
not use the two-stream schedule).  Per layer: the plan (BN, k-iterations per tile, tiles, grid, cluster size), the median time of
`reps` timed forwards, the issued MMA rate and the bytes the TMA ring moves from L2 into shared memory, computed from the plan.

    python tools/time_convs.py [fast] [json=PATH]
"""
import json, os, sys
import numpy as np, torch
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..')); sys.path.insert(0, ROOT)
import bench
import __graft_entry__

from oracle import synth
from ssd_keras_b200 import _ffi

BATCH = 32


def main():
    __graft_entry__.build()
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    fast = 'fast' in sys.argv[1:]
    out_json = next((a[5:] for a in sys.argv[1:] if a.startswith('json=')), None)
    prec = 'bf16' if fast else 'bf16x3'
    model = ssd_300((300, 300, 3), bench.N_CLASSES, mode='inference', scales=bench.SC300, divide_by_stddev=bench.STDDEV,
                    precision=prec)
    model.set_weights(bench._weights())
    x = torch.from_numpy(synth.synth_images(0, BATCH, 300, 300)).cuda()
    for _ in range(3):
        model.forward_device(x)
    torch.cuda.synchronize()
    convs = [s for s in model.specs if s.op in (_ffi.OP_CONV, _ffi.OP_HEAD)]
    model.set_timing(BATCH, True)
    reps, ms = 7, {s.name: [] for s in convs}
    for _ in range(reps):
        model.forward_device(x)
        torch.cuda.synchronize()
        for s in convs:
            ms[s.name].append(model.layer_ms(BATCH, s.name))
    model.set_timing(BATCH, False)
    props = torch.cuda.get_device_properties(0)
    rows, tot_ms, tot_bytes, tot_fl = [], 0.0, 0.0, 0.0
    for s in convs:
        p = model.layer_plan(BATCH, s.name)
        if p['kernel'] not in ('gemm', 'im2col_gemm'):
            continue
        taps = 1 if p['kernel'] == 'im2col_gemm' else s.kh * s.kw
        kiter = taps * p['kblocks']
        tiles = p['n_tiles_m'] * p['n_tiles_n']
        planes = 2 if p['split'] else 1
        stage = (128 * 64 * 2 + p['bn'] * 64 * 2) * planes
        l2_bytes = float(tiles) * kiter * stage
        issued = 2.0 * tiles * 128 * p['bn'] * (3 if p['split'] else 1) * kiter * 64
        t = float(np.median(ms[s.name]))
        rows.append({'layer': s.name, 'bn': p['bn'], 'stages': p['stages'], 'kiter': kiter, 'tiles': tiles, 'grid': p['grid'],
                     'cluster': p.get('cluster', 1), 'epilogue': p['epilogue'], 'ms': t, 'issued_tflops': issued / t / 1e9,
                     'l2_smem_gb': l2_bytes / 1e9, 'l2_smem_tbps': l2_bytes / t / 1e9})
        tot_ms += t; tot_bytes += l2_bytes; tot_fl += issued
    hdr = '%-12s %4s %3s %5s %6s %4s %3s %-6s %8s %8s %8s %8s' % ('layer', 'BN', 'stg', 'kiter', 'tiles', 'grid', 'cl', 'epi', 'ms',
                                                                  'TFLOP/s', 'L2->S GB', 'TB/s')
    print('%s, %d SMs, %s, batch %d, median of %d timed forwards (measured)' % (props.name, props.multi_processor_count, prec, BATCH, reps))
    print(hdr)
    for r in rows:
        print('%-12s %4d %3d %5d %6d %4d %3d %-6s %8.3f %8.1f %8.2f %8.2f' % (
            r['layer'], r['bn'], r['stages'], r['kiter'], r['tiles'], r['grid'], r['cluster'], r['epilogue'], r['ms'],
            r['issued_tflops'], r['l2_smem_gb'], r['l2_smem_tbps']))
    print('%-12s %50s %8.3f %8.1f %8.2f %8.2f' % ('total', '', tot_ms, tot_fl / tot_ms / 1e9, tot_bytes / 1e9, tot_bytes / tot_ms / 1e9))
    if out_json:
        with open(out_json, 'w') as f:
            json.dump({'gpu': props.name, 'precision': prec, 'layers': rows, 'total_ms': tot_ms}, f, indent=1)


if __name__ == '__main__':
    main()
