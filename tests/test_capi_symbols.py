"""CPU-side checks of the C-ABI boundary: the library builds/loads without a GPU driver and exports
every symbol include/otb200.h declares, and the ctypes binding has the header's signatures and struct layouts.
No compute calls."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def libpath():
    from opentransformer_b200 import build
    return build.build()


def _header_text():
    text = open(os.path.join(ROOT, 'include', 'otb200.h')).read()
    return re.sub(r'/\*.*?\*/|//[^\n]*', '', text, flags=re.S)


def _header_symbols():
    return sorted(set(re.findall(r'\b(otb_[a-z0-9_]+)\s*\(', _header_text())))


# What a C type is at the ABI, the granularity at which ctypes can get it wrong.
_C_KINDS = {'int': 'i32', 'int32_t': 'i32', 'uint32_t': 'u32', 'long long': 'i64', 'int64_t': 'i64', 'float': 'f32',
            'void': 'void'}
_C_STRUCTS = ('otb_beam_state', 'otb_mega_model')
_DECLARATOR = re.compile(r'(.*?)(\**)\s*(\w+)\s*(?:\[(\w+)\])?$', re.S)   # type, stars, name, array length


def _c_kind(type_text, stars, length=None, defines=None):
    base = ' '.join(w for w in re.findall(r'\w+', type_text) if w != 'const')
    if stars:
        return f'ptr:{base}' if base in _C_STRUCTS else 'pointer'
    if length is not None:
        return f'{base}[{defines.get(length, length)}]'
    return _C_KINDS[base]


def _parse_header():
    """-> ({function: (return kind, [argument kinds])}, {struct: [(field, kind)]}, {macro: value})."""
    text = _header_text()
    defines = dict(re.findall(r'^\s*#define\s+(\w+)\s+(\S+)', text, flags=re.M))
    text = re.sub(r'^\s*#.*$', '', text, flags=re.M)
    protos = {}
    for ret, name, params in re.findall(r'([\w\s*]+?)\b(otb_\w+)\s*\(([^()]*)\)\s*;', text):
        args = [] if params.strip() in ('', 'void') else [_DECLARATOR.match(p.strip()).groups() for p in params.split(',')]
        protos[name] = (_c_kind(ret, '*' in ret), [_c_kind(t, s) for t, s, _, _ in args])
    structs = {}
    for body, name in re.findall(r'typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;', text, flags=re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(';'))):
            first, *rest = decl.split(',')
            base, stars, field, length = _DECLARATOR.match(first.strip()).groups()
            fields.append((field, _c_kind(base, stars, length, defines)))
            for more in rest:                       # `const void *wqkv, *wo, ...`: the base type carries over
                _, stars, field, length = _DECLARATOR.match(more.strip()).groups()
                fields.append((field, _c_kind(base, stars, length, defines)))
        structs[name] = fields
    return protos, structs, defines


def _py_kind(t):
    from opentransformer_b200 import _lib
    if t is None:
        return 'void'
    if issubclass(t, ctypes._Pointer):
        return {_lib.BeamStateC: 'ptr:otb_beam_state', _lib.MegaModelC: 'ptr:otb_mega_model'}.get(t._type_, 'pointer')
    if issubclass(t, ctypes.Array):
        element = {_lib.MegaLayerC: 'otb_mega_layer'}[t._type_]
        return f'{element}[{t._length_}]'
    code = t._type_
    if code in ('P', 'z'):                          # c_void_p, c_char_p
        return 'pointer'
    if code == 'f':
        return 'f32'
    if code in 'bhilq':
        return f'i{8 * ctypes.sizeof(t)}'
    if code in 'BHILQ':
        return f'u{8 * ctypes.sizeof(t)}'
    raise AssertionError(f'no ABI kind for ctypes type {t}')


def test_library_loads_and_exports_every_declared_symbol(libpath):
    lib = ctypes.CDLL(libpath)
    syms = _header_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/otb200.h but not exported'


def test_python_binding_covers_the_header():
    """Every prototype in the header has a ctypes binding with the same return and argument kinds, in order.  A binding
    that drops an argument or passes c_int where the C function takes float still loads; it only goes wrong on the GPU."""
    from opentransformer_b200 import _lib, exported_symbols
    protos, _, _ = _parse_header()
    assert sorted(protos) == _header_symbols()
    assert exported_symbols() == _header_symbols()
    bad = []
    for name, want in sorted(protos.items()):
        res, args = _lib._SIGS[name]
        got = (_py_kind(res), [_py_kind(a) for a in args])
        if got != want:
            bad.append(f'{name}: header {want}, _SIGS {got}')
    assert not bad, 'ctypes signatures differ from include/otb200.h:\n' + '\n'.join(bad)


def test_ctypes_structs_match_the_header():
    """Field names, order and kinds of the ctypes mirrors of the header's structs, and the layer capacity."""
    from opentransformer_b200 import _lib
    _, structs, defines = _parse_header()
    for cname, mirror in (('otb_beam_state', _lib.BeamStateC), ('otb_mega_layer', _lib.MegaLayerC),
                          ('otb_mega_model', _lib.MegaModelC)):
        assert [(f, _py_kind(t)) for f, t in mirror._fields_] == structs[cname], f'{mirror.__name__} differs from {cname}'
    assert _lib.MEGA_MAX_LAYERS == int(defines['OTB_MEGA_MAX_LAYERS'])


def test_version_4_and_error_reporting(libpath):
    from opentransformer_b200 import _lib, ops
    lib = _lib.lib()
    assert lib.otb_version() == 4
    out = (ctypes.c_int * 6)()
    assert lib.otb_conv_geometry(1000, 80, *ops.CONV_SHIPPED, out) == 0 and out[0] == 499
    assert lib.otb_conv_geometry(3, 80, *ops.CONV_SHIPPED, out) != 0       # too short -> status, not abort
    assert b'otb_conv_geometry' in lib.otb_last_error()


def _capi_definitions():
    """-> [(name, body)] of every extern "C" otb_* function defined in csrc/capi.cu, comments stripped."""
    text = open(os.path.join(ROOT, 'opentransformer_b200', 'csrc', 'capi.cu')).read()
    text = re.sub(r'/\*.*?\*/|//[^\n]*', '', text, flags=re.S)
    text = text[text.index('extern "C" {'):]
    heads = list(re.finditer(r'^[A-Za-z][\w *]*?[ *](otb_\w+)\(', text, flags=re.M))
    return [(h.group(1), text[h.end():heads[i + 1].start() if i + 1 < len(heads) else len(text)]) for i, h in enumerate(heads)]


def test_every_entry_point_reports_under_its_own_name_and_calls_no_other():
    """One C entry point per operation: each otb_* definition reports its errors (fail / RET) under its own name only, and
    none forwards to another otb_* entry point, so the ABI does not grow wrappers that re-check and re-label errors."""
    defs = _capi_definitions()
    assert len(defs) == len(_header_symbols())
    bad = []
    for name, body in defs:
        bad += [f'{name} reports as {w}' for w in re.findall(r'\b(?:fail|RET)\(\s*([^,]+?)\s*,', body) if w != f'"{name}"']
        bad += [f'{name} calls {c}' for c in re.findall(r'\b(otb_\w+)\s*\(', body)]
    assert not bad, '\n'.join(bad)


def test_every_kernel_launches_through_one_helper():
    """Kernels are launched, and their shared-memory cap raised, only inside csrc/launch.cuh, so every kernel gets the same
    carve-out, cap and error handling.  No environment switch and no programmatic dependent launch anywhere."""
    csrc = os.path.join(ROOT, 'opentransformer_b200', 'csrc')
    bad = []
    for name in sorted(os.listdir(csrc)):
        text = open(os.path.join(csrc, name)).read()
        words = ['getenv', 'griddepcontrol', 'PDL_']
        if name != 'launch.cuh':
            words += ['<<<', 'cudaLaunchKernelEx', 'cudaFuncAttributeMaxDynamicSharedMemorySize']
        bad += [f'{name}: {w}' for w in words if w in text]
    assert not bad, 'outside the single launch path:\n' + '\n'.join(bad)


def test_conv_geometry_matches_reference_formula(libpath):
    from opentransformer_b200 import ops
    for T, F in [(1000, 80), (1000, 40), (777, 83), (90, 20), (7, 1)]:
        t1, f1, t2, f2 = ops.conv_geometry(T, F)
        assert t1 == (T - 3) // 2 + 1 and t2 == (t1 - 3) // 2 + 1          # frontend/conv.py:10-11, pad 0
        assert f1 == (F + 2 - 3) // 2 + 1 and f2 == (f1 + 2 - 3) // 2 + 1  # pad 1


def test_persistent_decode_host_arithmetic(libpath):
    """Host-only parts of the persistent decode entry points: workspace size (no GPU needed) and argument checks."""
    from opentransformer_b200 import _lib
    lib = _lib.lib()
    ws = lib.otb_decode_persistent_workspace
    base = ws(320, 6, 60, 32, 10, 4234)                 # benchmark geometry: 32 utterances x beam 10, 3 row groups
    assert base > 0
    groups, ldv = 3, (4234 + 31) // 32 * 32
    # dominated by the fp32 logits (128 rows per group) and the 16 fp32 feed-forward partial products per group
    assert base >= groups * 128 * ldv * 4 + 16 * groups * 128 * 256 * 4
    assert ws(640, 6, 60, 64, 10, 4234) > base          # more utterances -> more row groups
    assert ws(320, 6, 60, 32, 10, 8000) > base          # larger vocabulary -> larger logits buffer
    assert ws(320, 6, 60, 32, 17, 4234) == -1           # beam > 16 is not supported by the kernel
    assert ws(0, 6, 60, 32, 10, 4234) == -1
    assert lib.otb_set_decode_barrier(2) != 0 and b'otb_set_decode_barrier' in lib.otb_last_error()
    for kind in (1, 0, -1):
        assert lib.otb_set_decode_barrier(kind) == 0


def test_product_refuses_cpu_tensors(libpath):
    import torch
    from opentransformer_b200 import ops
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        ops.linear(torch.zeros(4, 64, dtype=torch.bfloat16), torch.zeros(8, 64, dtype=torch.bfloat16))


def test_state_dict_keys_match_reference_names():
    """Key names / shapes of the shipped transformer config (SURVEY.md 8b, probed from the reference)."""
    from opentransformer_b200.model import SpeechToText
    params = {'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
              'frontend': dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128,
                               kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                               front_end_layer_norm=False),
              'encoder': dict(d_model=256, n_heads=4, d_ff=2048, n_blocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                              ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False, concat_after=False,
                              activation='glu', relative_positional=False),
              'decoder': dict(vocab_size=4234, d_model=256, n_heads=4, d_ff=2048, memory_dim=256, n_blocks=1,
                              pos_dropout=0.0, slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0,
                              residual_dropout=0.1, activation='glu', normalize_before=False, concat_after=False,
                              share_embedding=True),
              'ctc_weight': 0.0, 'smoothing': 0.1}
    m = SpeechToText(params)
    enc, dec, fe = m.encoder.state_dict(), m.decoder.state_dict(), m.frontend.state_dict()
    assert tuple(enc['blocks.1.slf_attn.qvk_proj.weight'].shape) == (768, 256)
    assert tuple(enc['blocks.0.feed_forward.w_1.weight'].shape) == (4096, 256)
    assert tuple(dec['blocks.0.src_attn.vk_proj.weight'].shape) == (512, 256)
    assert tuple(fe['conv2.conv_layer.weight'].shape) == (128, 64, 3, 3)
    assert tuple(fe['output_layer.weight'].shape) == (256, 2560)
    assert dec['embedding.weight'].data_ptr() == dec['output_layer.weight'].data_ptr()   # tied
