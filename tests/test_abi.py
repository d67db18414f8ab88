"""The C-ABI library builds, loads and exports every symbol include/vt_b200.h declares (no compute calls)."""
import ctypes
import os
import re

from tests.conftest import ROOT


def test_library_exports_every_declared_symbol():
    from videotransformer_pytorch_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    hdr = open(os.path.join(ROOT, 'include', 'vt_b200.h')).read()
    declared = sorted(set(re.findall(r'^int\s+(vt_\w+)\s*\(', hdr, flags=re.M)))
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


def test_ctypes_param_structs_match_the_header(tmp_path):
    """Every ctypes Structure in _lib.py has the size and field offsets of its C twin in include/vt_b200.h."""
    import shutil
    import subprocess
    from videotransformer_pytorch_b200 import _lib
    if not shutil.which('gcc'):
        return
    pairs = {'vt_gemm_params': _lib.GemmParams, 'vt_ln_fwd_params': _lib.LnFwdParams, 'vt_ln_bwd_params': _lib.LnBwdParams,
             'vt_reduce_params': _lib.ReduceParams, 'vt_colsum_params': _lib.ColsumParams, 'vt_cast_params': _lib.CastParams,
             'vt_gather_cast_params': _lib.GatherCastParams, 'vt_gelu_params': _lib.GeluParams,
             'vt_attn_fwd_params': _lib.AttnFwdParams, 'vt_attn_bwd_params': _lib.AttnBwdParams,
             'vt_im2col_params': _lib.Im2colParams, 'vt_im2col_u8_params': _lib.Im2colU8Params, 'vt_hog_params': _lib.HogParams,
             'vt_pool_fwd_params': _lib.PoolFwdParams, 'vt_pool_bwd_params': _lib.PoolBwdParams,
             'vt_xattn_fwd_params': _lib.XattnFwdParams, 'vt_xattn_bwd_params': _lib.XattnBwdParams,
             'vt_maxpool_fwd_params': _lib.MaxpoolFwdParams, 'vt_maxpool_bwd_params': _lib.MaxpoolBwdParams,
             'vt_im2col3d_params': _lib.Im2col3dParams, 'vt_mvit_tokens_fwd_params': _lib.MvitTokensFwdParams,
             'vt_mvit_tokens_bwd_params': _lib.MvitTokensBwdParams, 'vt_mse_fwd_params': _lib.MseFwdParams,
             'vt_mse_bwd_params': _lib.MseBwdParams, 'vt_opt_params': _lib.OptParams,
             'vt_linear_small_params': _lib.LinearSmallParams, 'vt_linear_small_bwd_params': _lib.LinearSmallBwdParams,
             'vt_softmax_ce_params': _lib.SoftmaxCeParams, 'vt_scale_params': _lib.ScaleParams,
             'vt_im2col_u8_mix_params': _lib.Im2colU8MixParams,
             'vt_cls_rows_params': _lib.ClsRowsParams, 'vt_gather_cast_colsum_params': _lib.GatherCastColsumParams, 'vt_gelu_bwd_colsum_params': _lib.GeluBwdColsumParams}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "vt_b200.h")}"',
             'int main(void) {']
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
