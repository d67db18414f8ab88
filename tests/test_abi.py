"""The C ABI of include/vt_b200.h and its two mirrors: the library builds, loads and exports every symbol the header
declares (no compute calls); the ctypes structs and constants of _lib.py match the header; and the CPU kernel table of
tests/emu_kernels.py has every method of _lib.CudaKernels with the same parameters."""
import ctypes
import inspect
import os
import re

import pytest

from tests.conftest import ROOT

HEADER = os.path.join(ROOT, 'include', 'vt_b200.h')


def _declared_functions(hdr):
    return sorted(set(re.findall(r'^int\s+(vt_\w+)\s*\(', hdr, flags=re.M)))


def test_library_exports_every_declared_symbol():
    from videotransformer_pytorch_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    declared = _declared_functions(open(HEADER).read())
    assert len(declared) >= 15
    dll = ctypes.CDLL(path)
    for name in declared:
        assert hasattr(dll, name), f'{name} declared in vt_b200.h but not exported'
    assert sorted(_lib.EXPORTS) == declared
    assert dll.vt_version() == 1


def test_sass_is_hopper_native():
    import shutil
    import subprocess
    from videotransformer_pytorch_b200 import build
    if not shutil.which('cuobjdump'):
        return
    sass = subprocess.run(['cuobjdump', '-sass', build.build()], capture_output=True, text=True).stdout
    assert 'arch = sm_90a' in sass
    assert 'HGMMA' in sass          # wgmma.mma_async (GEMM)
    assert 'UTMALDG' in sass        # TMA loads (GEMM)
    assert 'HMMA.16816.F32.BF16' in sass   # mma.sync (flash attention)


def test_missing_library_fails_loudly(monkeypatch):
    import pytest
    from videotransformer_pytorch_b200 import _lib
    monkeypatch.setattr(_lib, '_dll', None)
    monkeypatch.setattr(_lib, 'LIB_PATH', '/nonexistent/libvt_b200.so')
    with pytest.raises(RuntimeError, match='no CPU / library fallback'):
        _lib.load_library()


def _struct_classes():
    """Each typedef struct of the header -> its ctypes class in _lib.py."""
    from videotransformer_pytorch_b200 import _lib as L
    return {
        'vt_gemm_params': L.GemmParams, 'vt_gemm_e4m3_params': L.GemmE4m3Params, 'vt_quant_rows_params': L.QuantRowsParams,
        'vt_ln_fwd_params': L.LnFwdParams, 'vt_ln_bwd_params': L.LnBwdParams, 'vt_reduce_params': L.ReduceParams,
        'vt_colsum_params': L.ColsumParams, 'vt_cast_params': L.CastParams, 'vt_gather_cast_params': L.GatherCastParams,
        'vt_gelu_params': L.GeluParams, 'vt_cls_rows_params': L.ClsRowsParams,
        'vt_gather_cast_colsum_params': L.GatherCastColsumParams, 'vt_gelu_bwd_colsum_params': L.GeluBwdColsumParams,
        'vt_attn_fwd_params': L.AttnFwdParams, 'vt_attn_bwd_params': L.AttnBwdParams,
        'vt_im2col_params': L.Im2colParams, 'vt_im2col_u8_params': L.Im2colU8Params, 'vt_col2im_params': L.Col2imParams,
        'vt_hog_params': L.HogParams, 'vt_pool_fwd_params': L.PoolFwdParams, 'vt_pool_bwd_params': L.PoolBwdParams,
        'vt_xattn_fwd_params': L.XattnFwdParams, 'vt_xattn_bwd_params': L.XattnBwdParams,
        'vt_maxpool_fwd_params': L.MaxpoolFwdParams, 'vt_maxpool_bwd_params': L.MaxpoolBwdParams,
        'vt_im2col3d_params': L.Im2col3dParams, 'vt_im2col3d_u8_params': L.Im2col3dU8Params,
        'vt_mvit_tokens_fwd_params': L.MvitTokensFwdParams, 'vt_mvit_tokens_bwd_params': L.MvitTokensBwdParams,
        'vt_mse_fwd_params': L.MseFwdParams, 'vt_mse_bwd_params': L.MseBwdParams, 'vt_opt_params': L.OptParams,
        'vt_linear_small_params': L.LinearSmallParams, 'vt_linear_small_bwd_params': L.LinearSmallBwdParams,
        'vt_softmax_ce_params': L.SoftmaxCeParams, 'vt_scale_params': L.ScaleParams, 'vt_topk_hits_params': L.TopkHitsParams,
        'vt_im2col_u8_mix_params': L.Im2colU8MixParams, 'vt_pos_resize_params': L.PosResizeParams,
        'vt_crop_desc': L.CropDesc, 'vt_resized_crop_params': L.ResizedCropParams, 'vt_jitter_desc': L.JitterDesc,
        'vt_color_jitter_params': L.ColorJitterParams, 'vt_randaug_desc': L.RandAugDesc,
        'vt_rand_augment_params': L.RandAugmentParams,
    }


def test_ctypes_param_structs_match_the_header(tmp_path):
    """Every struct the header declares has a ctypes Structure in _lib.py with its size and field offsets, and the
    exported names and constants of _lib.py are the header's."""
    import shutil
    import subprocess
    from videotransformer_pytorch_b200 import _lib
    hdr = open(HEADER).read()
    pairs = _struct_classes()
    assert set(pairs) == set(re.findall(r'typedef\s+struct\s*\{.*?\}\s*(vt_\w+)\s*;', hdr, flags=re.S))
    structs = {c for c in vars(_lib).values() if isinstance(c, type) and issubclass(c, ctypes.Structure)}
    assert structs <= set(pairs.values()) and len(set(pairs.values())) == len(pairs)
    assert sorted(_lib.EXPORTS) == _declared_functions(hdr)
    assert _lib.EPI == {n.lower(): int(v) for n, v in re.findall(r'\bVT_EPI_(\w+)\s*=\s*(\d+)', hdr)}
    assert _lib.RANDAUG_MAX_OPS == int(re.search(r'#define\s+VT_RANDAUG_MAX_OPS\s+(\d+)', hdr).group(1))
    if not shutil.which('gcc'):
        pytest.skip('gcc not available')
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            cf = 'in' if fname == 'inp' else fname
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {cf}));')
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', str(src), '-o', str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    got = {}
    for ln in out.splitlines():
        c, f, v = ln.split()
        got[(c, f)] = int(v)
    for cname, cls in pairs.items():
        assert got[(cname, 'size')] == ctypes.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert got[(cname, fname)] == getattr(cls, fname).offset, (cname, fname)


# CudaKernels members the CPU table does not mirror, and why
CUDA_ONLY = {
    'workspace': 'the per-stream device scratch buffer of the split-K GEMM; the emulation allocates as it goes',
    'name': "the table's label ('cuda' / 'emu'), which differs by design",
    'hog': 'the HOG targets are checked on the GPU against oracle/hog_oracle.py; no host-side path launches them',
}


def test_emu_table_mirrors_cuda_kernels():
    """EmuKernels has every public member of CudaKernels, and each method takes the same parameters (names, kinds and
    defaults), so a host-logic test runs the calls ops.py makes on the GPU."""
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200._lib import CudaKernels
    emu = EmuKernels()
    for name in sorted(n for n in dir(CudaKernels) if not n.startswith('_') and n not in CUDA_ONLY):
        assert hasattr(emu, name), f'EmuKernels has no {name}'
        member = getattr(CudaKernels, name)
        if callable(member):
            assert inspect.signature(getattr(EmuKernels, name)) == inspect.signature(member), name
