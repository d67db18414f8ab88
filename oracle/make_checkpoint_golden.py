"""Golden digests of the reference's pretrain_pth checkpoint remaps (its weight_init.py:107-314), for
tests/test_checkpoint_loaders.py.  Needs a checkout of the original project:

    python -m oracle.make_checkpoint_golden /path/to/VideoTransformer-pytorch

The synthetic checkpoints of the test are remapped by the reference's own functions; each resulting state dict is stored as
the SHA-256 of its keys, shapes, dtypes and bytes, so the test compares bit for bit without the reference present.
"""
import hashlib
import json
import os
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'checkpoint_remaps.json')


def digest(sd):
    """SHA-256 over the sorted keys and every tensor's shape, dtype and bytes"""
    h = hashlib.sha256()
    for k, v in sorted(sd.items()):
        h.update(f'{k}|{list(v.shape)}|{v.dtype}|'.encode())
        h.update(v.contiguous().numpy().tobytes())
    return h.hexdigest()


def reference_weight_init(ref):
    for name in ('matplotlib', 'matplotlib.pyplot', 'pytorch_lightning', 'pytorch_lightning.utilities'):
        sys.modules.setdefault(name, types.ModuleType(name))
    m = types.ModuleType('pytorch_lightning.utilities.distributed')
    m.rank_zero_only = lambda f: f
    sys.modules.setdefault('pytorch_lightning.utilities.distributed', m)
    sys.path.insert(0, ref)
    import importlib
    return importlib.import_module('weight_init')


def main(ref):
    sys.path.insert(0, ROOT)
    from tests import test_checkpoint_loaders as T

    W = reference_weight_init(ref)

    class Catch(torch.nn.Module):
        def load_state_dict(self, sd, strict=True):
            self.got = dict(sd)
            return torch.nn.modules.module._IncompatibleKeys([], [])

    out = {'remaps': {}}
    with tempfile.TemporaryDirectory() as tmp:
        for case in T.REMAP_CASES:
            for kind, make, fn, inner in (('vit', T._vit_image_checkpoint, W.init_from_vit_pretrain_, 'state_dict'),
                                          ('mae', T._mae_checkpoint, W.init_from_mae_pretrain_, 'model')):
                path = os.path.join(tmp, kind + '.pth')
                torch.save({inner: make()}, path)
                c = Catch()
                fn(c, path, *case, 2, 1)
                out['remaps'][T.case_id(kind, case)] = digest(c.got)
    sd = T._kinetics_checkpoint()
    W.replace_state_dict(sd)
    out['kinetics'] = digest(sd)
    with open(OUT, 'w') as fh:
        json.dump(out, fh, indent=0, sort_keys=True)
    print(f'wrote {OUT}')


if __name__ == '__main__':
    main(sys.argv[1])
