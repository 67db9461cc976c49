"""CPU-only checks of the host side: state_dict contract, config translation, the C-ABI
library (loads, exports every declared symbol, argument validation without touching a GPU),
weight folding/packing, and that the product never routes through the oracle."""
import os
import re

import pytest
import torch

from conftest import ROOT, GOLDEN_FULL
from openglue_b200 import _cabi
from openglue_b200.packing import pack_weights
from openglue_b200.superglue import SuperGlue
from openglue_b200.synthetic import default_config, synthetic_state_dict
from oracle import superglue_oracle as O
from packed_emulation import forward_packed


def test_library_exports_every_header_symbol():
    header = open(os.path.join(ROOT, 'include', 'openglue_b200.h')).read()
    declared = set(re.findall(r'\b(og_[a-z0-9_]+)\s*\(', header))
    declared -= {'og_status', 'og_config'}
    lib = _cabi.lib()
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in the header but not exported'
    assert declared == set(_cabi.SYMBOLS), declared ^ set(_cabi.SYMBOLS)
    assert lib.og_version() == 100


def test_abi_struct_sizes_match_header():
    # og_config: 5 + 8 ints, int, float, float, int, int = 18 * 4 bytes
    import ctypes as C
    assert C.sizeof(_cabi.OgConfig) == 18 * 4
    assert C.sizeof(_cabi.OgLinearArgs) == 192


def test_argument_validation_without_gpu():
    lib = _cabi.lib()
    cfg = _cabi.make_config(default_config())
    assert lib.og_workspace_bytes(cfg, 0, 10, 10) < 0
    assert b'positive' in lib.og_last_error()
    bad = _cabi.make_config(default_config(descriptor_dim=30, num_heads=4))
    assert lib.og_packed_weight_floats(bad) < 0
    assert lib.og_superglue_forward(cfg, None, None, None, 1, 8, 8, None, None, None, None, None, None, None, None, None, None,
                                    None, None, None, None, None, 0, None) == -1     # OG_EINVAL, no CUDA call made
    assert lib.og_workspace_bytes(cfg, 2, 100, 3000) > 0                             # wide rows: several warps share a row
    assert lib.og_workspace_bytes(cfg, 2, 100, 9000) < 0 and b'8192' in lib.og_last_error()   # the documented limit


def test_state_dict_contract_matches_reference_layout(golden):
    for name in ['tiny_flat', 'tiny_offset_s6']:
        fx = golden(name)
        model = SuperGlue(dict(fx['config']))
        ours = model.state_dict()
        assert list(ours.keys()) == list(fx['state_dict'].keys())
        for k, v in fx['state_dict'].items():
            assert tuple(ours[k].shape) == tuple(v.shape), k
        model.load_state_dict(fx['state_dict'], strict=True)
    full = SuperGlue(default_config())
    assert len(full.state_dict()) == 333                       # SURVEY.md section 8(b)
    assert sum(p.numel() for p in full.parameters()) == 11_957_249


def test_unsupported_options_raise():
    cfg = default_config()
    cfg['attention_gnn']['attention'] = 'linear'
    with pytest.raises(ValueError):
        SuperGlue(cfg)
    cfg = default_config()
    cfg['positional_encoding']['encoder_name'] = 'Nope'
    with pytest.raises(NameError):
        SuperGlue(cfg)
    model = SuperGlue(default_config(descriptor_dim=32, num_stages=1)).eval()
    data = {'keypoints0': torch.zeros(1, 4, 2), 'keypoints1': torch.zeros(1, 4, 2)}
    with pytest.raises(RuntimeError, match='no CPU path'):
        model(data)


def test_weights_version_sees_every_kind_of_weight_change():
    """The fingerprint that keys the packed weights and the captured graphs changes with each way a weight can change,
    including tensors replaced by assignment (a new Parameter, buffer or submodule object), and only then."""
    cfg = default_config(descriptor_dim=64, num_stages=1, num_iters=5)
    model = SuperGlue(cfg).eval()
    model.load_state_dict(synthetic_state_dict(cfg))
    layer = model.attention_gnn.layers[0].module

    def scale_in_place():
        with torch.no_grad():
            model.linear_proj.weight.mul_(1.01)

    changes = [
        scale_in_place,
        lambda: model.load_state_dict(synthetic_state_dict(cfg, seed=1)),
        lambda: setattr(model.dustbin_score, 'data', model.dustbin_score.data + 1),
        lambda: setattr(model.linear_proj, 'weight', torch.nn.Parameter(model.linear_proj.weight.detach() * 2)),
        lambda: setattr(layer.fc[2], 'running_mean', layer.fc[2].running_mean + 1),
        lambda: setattr(layer.mha, 'in_proj_q', torch.nn.Conv1d(64, 64, kernel_size=1)),
    ]
    seen = [model._weights_version()]
    assert model._weights_version() == seen[0]
    for change in changes:
        change()
        v = model._weights_version()
        assert v not in seen
        assert model._weights_version() == v
        seen.append(v)


@pytest.mark.parametrize('name', GOLDEN_FULL)
def test_weight_folding_and_packing(golden, name):
    """packed weights + the kernel schedule (torch emulation, fp64) == oracle fp64."""
    fx = golden(name)
    cfg = _cabi.make_config(fx['config'])
    packed64 = pack_weights(fx['state_dict'], fx['config'], cfg, dtype=torch.float64)
    got = forward_packed(packed64, fx['config'], cfg, fx['data'])
    assert (got['scores'] - fx['scores_f64']).abs().max() < 5e-6     # the reference keeps log_a/log_b/norm in fp32
    ref = O.run(fx['state_dict'], fx['config'], fx['data'], dtype=torch.float64)
    assert (got['context_descriptors0'] - ref['context_descriptors0']).abs().max() < 1e-10
    # and the fp32 packing is the rounding of the fp64 one
    packed = pack_weights(fx['state_dict'], fx['config'], cfg)
    assert packed.dtype == torch.float32
    assert (packed.double() - packed64).abs().max() <= packed64.abs().max() * 2 ** -23


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'openglue_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle', text, re.M), f
                assert '/root/reference' not in text, f


def test_tensor_core_kernels_are_hopper_native_and_address_shared_memory_directly():
    """Static check of the built library (cuobjdump, no GPU): every kernel that issues warpgroup MMAs (HGMMA in SASS) stages its
    operands with TMA, and none of them contains a generic LD.E / ST.E - the dynamic shared-memory block is aligned as an offset
    from the __shared__ symbol (tc::align_smem_1024); aligning it through uintptr_t hides the address space from the compiler."""
    import collections
    import re
    import shutil
    import subprocess
    from openglue_b200 import _cabi
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    out = subprocess.run([tool, '-sass', _cabi.LIB_PATH], capture_output=True, text=True).stdout
    hist, cur = {}, None
    for line in out.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = hist.setdefault(m.group(1), collections.Counter())
            continue
        m = re.match(r'\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
        if m and cur is not None:
            cur[m.group(1).split('.')[0] + ('.E' if m.group(1).startswith(('LD.E', 'ST.E')) else '')] += 1
    tc = {k: c for k, c in hist.items() if c['HGMMA'] > 0}
    assert len(tc) >= 5                                    # GEMM (tf32 / fp16 operands) and attention (tf32 Dh 32 / 64, fp16)
    for name, c in tc.items():
        assert c['LD.E'] == 0 and c['ST.E'] == 0, (name, c['LD.E'], c['ST.E'])
        assert c['UTMALDG'] > 0, name                      # operands staged by TMA
    attn = [c for k, c in tc.items() if 'attention_sm90_kernel' in k]
    assert len(attn) == 3 and all(c['MUFU'] >= 32 for c in attn)


def test_sinkhorn_kernels_are_the_planned_instantiations_without_spills():
    """Static check of the built library (cuobjdump, no GPU; OG_LIB names another build): it holds exactly the five forward and
    five backward cooperative Sinkhorn instantiations sinkhorn_plan can select, and none touches local memory (STL / LDL:
    spills) - the V = 16 forms sit within a few registers of the 255 limit.  Uniform and padded batches run the same kernels
    (the per-pair lengths are a runtime argument), so every Sinkhorn, attention, match and encoder-input kernel is one of the
    planned instantiations, with no second, padded form beside it."""
    import re
    import shutil
    import subprocess
    from openglue_b200 import _cabi
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    path = os.environ.get('OG_LIB') or _cabi.LIB_PATH
    assert os.path.exists(path), f'library not built: {path}'
    res = subprocess.run([tool, '-sass', path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    funcs, cur = {}, None
    for line in res.stdout.splitlines():
        m = re.match(r'\s*Function : _ZN2og(?:15sinkhorn_kernel|19sinkhorn_bwd_kernel)ILi(\d+)ELi(\d+)ELi(\d+)EEEvNS_\d+([A-Za-z]\w*)E$', line)
        if m:
            cur = funcs.setdefault((m.group(4),) + tuple(int(g) for g in m.group(1, 2, 3)), [])
            continue
        if re.match(r'\s*Function : ', line):
            cur = None
            continue
        m = re.match(r'\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P(?:\d+|T)\s+)?([A-Z0-9_.]+)', line)
        if m and cur is not None:
            cur.append(m.group(1).split('.')[0])
    bands = [(4, 1), (4, 2), (8, 2), (16, 2), (16, 4)]
    fwd = {('SinkArgs', v, w, 1 if w == 4 else 2) for v, w in bands}
    bwd = {('SinkBwdArgs', v, w, 1 if v == 16 else 2) for v, w in bands}
    assert set(funcs) == fwd | bwd, sorted(funcs)
    for name, ops in funcs.items():
        assert 'STL' not in ops and 'LDL' not in ops, name

    def kernel(mangled):                                   # _ZN2og<len><name>[I<L{i,b}<value>E>...E]E...: (name, template values)
        m = re.match(r'_ZN2og(\d+)', mangled)
        name = mangled[m.end():m.end() + int(m.group(1))]
        targs = re.match(r'I((?:L[ib]\d+E)+)E', mangled[m.end() + len(name):])
        return name, tuple(int(v) for v in re.findall(r'\d+', targs.group(1))) if targs else ()
    operators = {kernel(k) for k in re.findall(r'^\s*Function : (_ZN2og\S+)$', res.stdout, re.M)}
    operators = {k for k in operators if re.match(r'(sinkhorn|attention|match|kenc)_', k[0])}
    planned = ({('sinkhorn_kernel', k[1:]) for k in fwd} | {('sinkhorn_bwd_kernel', k[1:]) for k in bwd} |
               {('sinkhorn_resident_kernel', (v, w, 16 // v)) for v, w in [(4, 1), (4, 2), (8, 2)]} |
               {('attention_sm90_kernel', k) for k in [(32, 0), (64, 0), (64, 1)]} |
               {('attention_simt_kernel', (dh,)) for dh in (8, 16, 32, 64)} |
               {(f'match_{op}_kernel', ()) for op in ('rowmax', 'colmax', 'colreduce', 'finalize', 'compact')} |
               {('sinkhorn_consts_kernel', ()), ('kenc_input_kernel', ())})
    assert operators == planned, sorted(operators ^ planned)


def test_bench_work_accounting_reproduces_the_survey_table():
    """bench.py's algorithmic FLOP / byte formulas against the values SURVEY.md (section 8d, Appendix B) states for the BASELINE
    configurations - the numerators of `roofline.achieved` and of the judge's own check."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('og_bench', os.path.join(ROOT, 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    rel = lambda a, b: abs(a - b) / b
    # (n, m, d, stages, S, T) -> (F_total, F_attn, Q_sink GB)
    table = {'C1': ((512, 512, 256, 9, 1, 20), (3.418e10, 9.66e9, 0.0221)),
             'C2': ((1024, 1024, 256, 9, 1, 100), (8.796e10, 3.865e10, 0.4245)),
             'C3': ((2048, 2048, 256, 9, 1, 100), (2.543e11, 1.546e11, 1.696)),
             'C5': ((4096, 1024, 128, 18, 6, 50), (3.035e11, 2.416e11, 0.857))}
    for name, ((n, m, d, stages, s, t), (ftot, fattn, qs)) in table.items():
        fl = bench.flops_per_pair(n, m, d, stages, s)
        assert rel(fl['total'], ftot) < 2e-3 and rel(fl['attn'], fattn) < 2e-3, (name, fl)
        assert rel(bench.sinkhorn_bytes_per_pair(n, m, t) / 1e9, qs) < 3e-3, name
        wl = bench.BASELINE_CONFIGS[name]
        assert (wl['n'], wl['m'], wl['cfg']['descriptor_dim'], wl['cfg']['num_stages'], wl['cfg']['num_iters']) == (n, m, d, stages, t)
    assert bench.BASELINE_CONFIGS['C4']['n'] == 2048 and bench.BASELINE_CONFIGS['C4']['cfg']['num_iters'] == 100
