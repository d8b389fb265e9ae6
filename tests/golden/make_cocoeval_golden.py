#!/usr/bin/env python
"""The twelve summary lines that the reference's ssd300_evaluation_COCO.ipynb stores as the output of its last evaluation cell
(pycocotools' COCOeval.summarize on val2017).  Copies those lines, data only, to tests/golden/ref_cocoeval_summary.txt.
Build container only."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')


def main():
    with open(os.path.join(ROOT, 'ssd300_evaluation_COCO.ipynb')) as f:
        nb = json.load(f)
    lines = []
    for cell in nb['cells']:
        for out in cell.get('outputs', []):
            lines += [l for l in ''.join(out.get('text', '')).split('\n') if l.startswith(' Average ')]
    assert len(lines) == 12, lines
    with open(os.path.join(HERE, 'ref_cocoeval_summary.txt'), 'w') as f:
        f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
