"""The C ABI of include/vt_attn_maps.h and its mirrors: the library exports every symbol the header declares (no compute
calls); the ctypes structs and export list of attn_maps_lib match the header; and the CPU table of
tests/emu_attention_maps.py has every method of attn_maps_lib.CudaAttnMapKernels with the same parameters."""
import ctypes
import inspect
import os
import re
import shutil
import subprocess

import pytest

from tests.conftest import ROOT

HEADER = os.path.join(ROOT, 'include', 'vt_attn_maps.h')


def test_library_exports_every_declared_symbol():
    from videotransformer_pytorch_b200 import attn_maps_lib, build
    hdr = open(HEADER).read()
    declared = sorted(set(re.findall(r'^int\s+(vt_\w+)\s*\(', hdr, flags=re.M)))
    assert declared == sorted(attn_maps_lib.EXPORTS) == ['vt_attn_cls_probs', 'vt_attn_mass_mask']
    dll = ctypes.CDLL(build.build())
    for name in declared:
        assert hasattr(dll, name), f'{name} declared in vt_attn_maps.h but not exported'


def test_ctypes_param_structs_match_the_header(tmp_path):
    from videotransformer_pytorch_b200 import attn_maps_lib as L
    hdr = open(HEADER).read()
    pairs = {'vt_attn_cls_probs_params': L.AttnClsProbsParams, 'vt_attn_mass_mask_params': L.AttnMassMaskParams}
    assert set(pairs) == set(re.findall(r'typedef\s+struct\s*\{.*?\}\s*(vt_\w+)\s*;', hdr, flags=re.S))
    structs = {c for c in vars(L).values() if isinstance(c, type) and issubclass(c, ctypes.Structure)}
    assert structs == set(pairs.values())
    if not shutil.which('gcc'):
        pytest.skip('gcc not available')
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', str(src), '-o', str(exe)])
    got = {}
    for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        c, f, v = ln.split()
        got[(c, f)] = int(v)
    for cname, cls in pairs.items():
        assert got[(cname, 'size')] == ctypes.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert got[(cname, fname)] == getattr(cls, fname).offset, (cname, fname)


def test_emu_table_mirrors_cuda_table():
    from tests.emu_attention_maps import EmuAttnMapKernels
    from videotransformer_pytorch_b200.attn_maps_lib import CudaAttnMapKernels
    for name in sorted(n for n in dir(CudaAttnMapKernels) if not n.startswith('_')):
        assert hasattr(EmuAttnMapKernels, name), f'EmuAttnMapKernels has no {name}'
        member = getattr(CudaAttnMapKernels, name)
        if callable(member):
            assert inspect.signature(getattr(EmuAttnMapKernels, name)) == inspect.signature(member), name
