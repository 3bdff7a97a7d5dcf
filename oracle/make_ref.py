"""TEST / BASELINE INFRASTRUCTURE -- recipe that copies the UNMODIFIED Python reference (NVIDIA/vid2vid) into the git-ignored
oracle/_ref/, so that it travels with a working tree to a machine without the reference tree.

    python oracle/make_ref.py      # also run by __graft_entry__.build()

The reference tree is V2V_REFERENCE_SRC if set, else a checkout named `reference` next to this repository or next to one of
its parent directories (found by its models/vid2vid_model_G.py).  Copies only the importable Python modules of the hot path
(models/, util/, options/ -- no CUDA sources, images, scripts or checkpoints).  Used by bench.py `--impl reference` /
`cpu_baseline` to time the reference's own Vid2VidModelG.inference on the host cores (kind "reference"), and by the GPU test
that swaps vid2vid_b200.networks into the reference's Vid2VidModelG (INTEGRATION.md section 2).  Without a reference tree
nothing is copied: that test skips and the CPU arm times the oracle port (kind "port")."""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, '_ref')


def _is_reference(d):
    return os.path.isfile(os.path.join(d, 'models', 'vid2vid_model_G.py'))


def find_reference():
    """The reference tree to copy from, or None."""
    src = os.environ.get('V2V_REFERENCE_SRC')
    if src:
        return src if _is_reference(src) else None
    d = os.path.dirname(HERE)                       # the repository root
    while True:
        parent = os.path.dirname(d)
        cand = os.path.join(parent, 'reference')
        if _is_reference(cand):
            return cand
        if parent == d:
            return None
        d = parent


def make():
    src = find_reference()
    if src is None:
        return None
    n = 0
    for top in ('models', 'util', 'options'):
        for root, dirs, files in os.walk(os.path.join(src, top)):
            rel = os.path.relpath(root, src)
            for f in files:
                if f.endswith('.py'):
                    os.makedirs(os.path.join(DST, rel), exist_ok=True)
                    shutil.copyfile(os.path.join(root, f), os.path.join(DST, rel, f))
                    n += 1
    with open(os.path.join(DST, 'SOURCE.txt'), 'w') as f:
        f.write('copied unmodified by oracle/make_ref.py (%d files)\n' % n)
    return DST


if __name__ == '__main__':
    dst = make()
    print(dst or 'no reference tree found (set V2V_REFERENCE_SRC)', file=sys.stdout if dst else sys.stderr)
