"""FP8 LM weights (weight_dtype='fp8') on the H100: every FP8 decode-GEMM instance against float64, the scoring forward
against the fp16 forward of the dequantized weights, and the equalities of the fp16 path, which hold within FP8.

References.  A row reads back as code * scale, exact in float64 (a 4-bit code times an fp32 scale), so the float64 GEMM of
the activations with the dequantized rows is scale[n] * sum_k code x.  The kernels unpack each code exactly to fp16, the
products code x are exact in fp32, the fixed-order fp32 sum meets (K - 1) 2^-24 sum |code x| and the one fp32 product with
the scale adds 2^-24 of the result: the checks of tests/test_gpu_kernels_f64 and tests/test_gpu_decode_f64 run unchanged
on those references, with `gemm64` widened by that one rounding where the weights are FP8 (float64 here) and the fp16 half
ulp added by the same checkers where the output is fp16.  Each check prints its worst fraction of the bound.

The decode-GEMM sweep is test_decode_gemms_match_float64's (rows 2, 12, 24, 40, 64, 80, 200: NT 1, 2, 4, 8, 8 on
lm_gemm_fp8_kernel, NPAD 128 / 256 on lm_gemm_wide_fp8_kernel; sin and rope; ACB_LM_FT32 on and off).  The prompt-pass
(QKV_PF, QKV_PF_ROPE and the paged admission's F32) and CROSSKV instances run through test_gpu_decode_f64's prefill and
decode-step probes.  The equalities are existing tests of the fp16 path run with every LMModel built as FP8."""
import ctypes as C
import functools

import pytest
import torch

from audiocraft_b200 import _lib, synth
from audiocraft_b200.lm import LMModel
from tests import test_gpu_decode_f64 as D
from tests import test_gpu_kernels_f64 as K

U = 2.0 ** -24
LAYER_MATRICES = ('w_qkv', 'w_o', 'w_cq', 'w_ckv', 'w_co', 'w_ff1', 'w_ff2')


def dequant64(m):
    """m's weights with every FP8 matrix as float64 code * scale (exact); the other tensors as stored."""
    w = dict(m._w)
    for n in LAYER_MATRICES:
        if w[n] is not None:
            w[n] = w[n].double() * w['s' + n[1:]].double().unsqueeze(-1)
    return w


class RefView:
    """The FP8 model with `_w` replaced by its float64 dequantized weights for the references; everything else is the model
    (the handle, buffers and methods keep reading the stored codes and scales)."""

    def __init__(self, m):
        object.__setattr__(self, '_m', m)
        object.__setattr__(self, '_w', dequant64(m))

    def __getattr__(self, name):
        return getattr(self._m, name)

    def __setattr__(self, name, value):
        setattr(self._m, name, value)


def _gemm64_fp8(orig):
    @functools.wraps(orig)
    def gemm64(a, w):
        v64, bnd = orig(a, w)
        if w.dtype == torch.float64:   # FP8 rows: one more fp32 rounding, of the scale product
            bnd = bnd + U * (v64.abs() + bnd)
        return v64, bnd
    return gemm64


@pytest.fixture
def fp8_refs(monkeypatch):
    monkeypatch.setattr(K, 'gemm64', _gemm64_fp8(K.gemm64))
    monkeypatch.setattr(D, 'gemm64', _gemm64_fp8(D.gemm64))

    def probe(name, pe, cross, prefix=False, seed=7):
        cfg, sd0, m = _probe_fp16_args(name, pe, cross, prefix, seed)
        return cfg, sd0, RefView(m)
    monkeypatch.setattr(D, '_probe', probe)


_PROBE = D._probe


def _probe_fp16_args(name, pe, cross, prefix, seed):
    """test_gpu_decode_f64._probe's model, built with FP8 weights."""
    orig = LMModel.__init__
    try:
        LMModel.__init__ = lambda self, sd, cfg, cp=None, fu=None, device='cuda', weight_dtype='fp8': \
            orig(self, sd, cfg, cp, fu, device, 'fp8')
        cfg, sd0, m = _PROBE(name, pe, cross, prefix, seed)
    finally:
        LMModel.__init__ = orig
    assert m.weight_dtype == 'fp8'
    return cfg, sd0, m


@pytest.fixture
def all_fp8(monkeypatch):
    """Every LMModel built during the test stores FP8 weights (whatever weight_dtype its caller passes)."""
    orig = LMModel.__init__
    built = []

    def init(self, state_dict, cfg, condition_provider=None, fuser=None, device='cuda', weight_dtype='fp16'):
        orig(self, state_dict, cfg, condition_provider, fuser, device, 'fp8')
        built.append(self)
    monkeypatch.setattr(LMModel, '__init__', init)
    yield built
    assert built and all(m.weight_dtype == 'fp8' for m in built)


# ----------------------------------------------------------------------------- decode GEMMs against float64

@pytest.mark.gpu
@pytest.mark.parametrize('name,pe,ft32', [
    ('lm_mini', 'sin', None), ('lm_mini', 'rope', None), ('lm_medium_2l', 'sin', None), ('lm_medium_2l', 'rope', None),
    ('lm_large_2l', 'sin', None), ('lm_large_2l', 'rope', None), ('lm_medium_2l', 'sin', '0')],
    ids=['lm_mini-sin', 'lm_mini-rope', 'lm_medium_2l-sin', 'lm_medium_2l-rope', 'lm_large_2l-sin', 'lm_large_2l-rope',
         'lm_medium_2l-sin-ft16'])
def test_fp8_decode_gemms_match_float64(monkeypatch, fp8_refs, name, pe, ft32):
    """Every lm_gemm_fp8_kernel / lm_gemm_wide_fp8_kernel instance of the decode step through acb_lm_debug_gemms: each
    layer's K / V at the step's position, the last layer's q32 and GELU output, the FF2 partial sums (each K slice scaled
    before it is stored) against scale[n] * sum_k code x in float64."""
    if ft32 is None:
        monkeypatch.delenv('ACB_LM_FT32', raising=False)
    else:
        monkeypatch.setenv('ACB_LM_FT32', ft32)
    cfg0, sd0 = K._synth(name, (), True, 7)
    cfg = dict(cfg0, positional_embedding=pe)
    sd = K.probe_state_dict(cfg, sd0, ('self_attn.out_proj.weight', 'cross_attention.out_proj.weight'), False)
    for li in range(cfg['num_layers']):
        p = f'transformer.layers.{li}.cross_attention.in_proj_weight'
        sd[p] = sd[p].clone()
        sd[p][:cfg['dim']] = 0
    m = LMModel(sd, cfg, None, None, weight_dtype='fp8')
    assert m._w['w_qkv'].dtype == torch.float8_e4m3fn and m._w['s_qkv'].shape == (cfg['num_layers'], 3 * cfg['dim'])
    ref = RefView(m)
    rows_list = K.DECODE_ROWS if ft32 is None else (2, 12, 24, 40)
    for i, rows in enumerate(rows_list):
        K._decode_pass(ref, cfg, rows, 300 - rows, 100 + i, f'fp8 {name} {pe}' + (' ft16' if ft32 else ''))


PASS_CASES = [c for c in D.PREFILL_CASES if c[0] in ('contiguous-rope-B1', 'contiguous-sin-B2-cross',
                                                       'contiguous-sin_rope-B3-cross', 'paged-rope-P0-F33',
                                                       'melody-sin_rope-P64')]


@pytest.mark.gpu
@pytest.mark.parametrize('case', PASS_CASES, ids=[c[0] for c in PASS_CASES])
def test_fp8_prefill_passes_match_float64(fp8_refs, case):
    """EPI_QKV_PF / EPI_QKV_PF_ROPE (contiguous prompt and prefix passes) and the paged admission pass's EPI_F32 on FP8
    weights, through test_gpu_decode_f64's prefill probe."""
    D.test_prefill_passes_match_float64(case)


STEP_CASES = [c for c in D.GEN_CASES if c[0] in ('mini-sin-cross-B1-text65', 'medium-sin-cross-B6-text32', 'large-rope-B6')]


@pytest.mark.gpu
@pytest.mark.parametrize('case', STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_fp8_decode_step_and_cross_kv_match_float64(fp8_refs, case):
    """The decode step on FP8 weights through test_gpu_decode_f64's step probe, including EPI_CROSSKV at acb_lm_begin."""
    D.test_generate_step_matches_float64(case)


# ----------------------------------------------------------------------------- scoring forward

def _dequant_state_dict(m, sd):
    """sd with every per-layer matrix replaced by its fp16 dequantized value fp16(fp32(code * scale))."""
    d, out = m.dim, dict(sd)
    w = m._w
    deq = {n: (w[n].float() * w['s' + n[1:]].unsqueeze(-1)).half().cpu() for n in LAYER_MATRICES if w[n] is not None}
    for li in range(m.num_layers):
        p = f'transformer.layers.{li}.'
        out[p + 'self_attn.in_proj_weight'] = deq['w_qkv'][li]
        out[p + 'self_attn.out_proj.weight'] = deq['w_o'][li]
        out[p + 'linear1.weight'] = deq['w_ff1'][li]
        out[p + 'linear2.weight'] = deq['w_ff2'][li]
        if m.cross_attention:
            out[p + 'cross_attention.in_proj_weight'] = torch.cat([deq['w_cq'][li], deq['w_ckv'][li]])
            out[p + 'cross_attention.out_proj.weight'] = deq['w_co'][li]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('name,pe,B,S,Tt,P', [('lm_mini', 'sin', 3, 65, 33, 0), ('lm_mini', 'rope', 2, 130, None, 0),
                                             ('lm_medium_2l', 'sin_rope', 1, 64, 65, 0),
                                             ('lm_mini_melody', 'rope', 2, 63, None, 9)])
def test_fp8_forward_equals_fp16_forward_of_dequantized_weights(name, pe, B, S, Tt, P):
    """acb_lm_forward on FP8 weights dequantizes each layer to fp16(code * scale) in its workspace and runs the fp16 GEMMs
    on it, so its logits are bit for bit those of an fp16 model holding the dequantized weights (whose every stage
    tests/test_gpu_kernels_f64 checks against float64); the last layer's dequantized matrices are read back from the
    workspace and compared with fp16(fp32(code * scale)) bit for bit."""
    cross = Tt is not None
    cfg0, sd0 = K._synth(name, (), cross, 7)
    cfg = dict(cfg0, positional_embedding=pe)
    m8 = LMModel(sd0, cfg, None, None, weight_dtype='fp8')
    m16 = LMModel(_dequant_state_dict(m8, sd0), cfg, None, None)
    g = torch.Generator().manual_seed(B * 100 + S)
    d = cfg['dim']
    seq = torch.randint(0, cfg['card'] + 1, (B, cfg['n_q'], S), generator=g)
    kw = {}
    if cross:
        kw['cross_attention_src'] = torch.randn(B, Tt, d, generator=g) * 0.5
    if P:
        kw['prefix'] = torch.randn(B, P, d, generator=g) * 0.5
    a, b = m8.forward(seq, **kw), m16.forward(seq, **kw)
    assert torch.equal(a, b), f'{name} {pe}: FP8 forward differs from the fp16 forward of the dequantized weights'

    # the workspace: the fp16 layout of test_gpu_kernels_f64.fwd_layout, then one layer's seven matrices
    cfg_c, lay = m8._config(), K.fwd_layout(cfg, B, P, S, Tt or 0)
    n = m8._lib.acb_lm_forward_workspace_bytes(C.byref(cfg_c), B, P, S, Tt or 0)
    ffn, L = int(cfg['hidden_scale'] * d), cfg['num_layers']
    shapes = [('w_qkv', 3 * d, d), ('w_o', d, d)] + ([('w_cq', d, d), ('w_ckv', 2 * d, d), ('w_co', d, d)] if cross else []) + \
        [('w_ff1', ffn, d), ('w_ff2', d, ffn)]
    assert n == lay['total'] + sum((r * c * 2 + 255) // 256 * 256 for _, r, c in shapes), 'one layer of fp16 matrices more'
    seq_d = seq.cuda()
    ws = torch.full((n,), 0xFF, dtype=torch.uint8, device='cuda')
    logits = torch.empty((B, cfg['n_q'], S, cfg['card']), device='cuda')
    cr = kw['cross_attention_src'].cuda() if cross else None
    pf = kw['prefix'].cuda() if P else None
    _lib.check(m8._lib.acb_lm_forward(C.byref(cfg_c), C.byref(m8._weights()), _lib.ptr(seq_d), _lib.ptr(cr), _lib.ptr(pf), B, P,
                                      S, Tt or 0, _lib.ptr(logits), _lib.ptr(ws), n, _lib.stream()), 'lm_forward')
    torch.cuda.synchronize()
    assert torch.equal(logits, a)
    off, w = lay['total'], m8._w
    for nm, r, c in shapes:
        got = ws[off:off + r * c * 2].view(torch.float16).view(r, c)
        want = (w[nm][L - 1].float() * w['s' + nm[1:]][L - 1].unsqueeze(-1)).half()
        assert torch.equal(got, want), f'{nm}: the workspace copy is not fp16(code * scale)'
        off += (r * c * 2 + 255) // 256 * 256


# ----------------------------------------------------------------------------- equalities that hold within FP8

@pytest.mark.gpu
@pytest.mark.parametrize('name', ['lm_mini', 'lm_medium_2l'])
def test_fp8_generate_is_reproducible_and_keeps_the_launch_count(name):
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=3)
    m16, m8 = LMModel(sd, cfg, None, None), LMModel(sd, cfg, None, None, weight_dtype='fp8')
    assert m8.weight_bytes_per_step < 0.6 * m16.weight_bytes_per_step
    cross = torch.randn(4, 9, cfg['dim']) * 0.5
    outs = []
    for m in (m8, m8, m16):
        torch.manual_seed(11)
        outs.append(m.generate(num_samples=2, max_gen_len=40, cross_attention_src=cross, top_k=50))
    assert torch.equal(outs[0], outs[1]), 'two FP8 generate calls with the same seed differ'
    assert m8.launches_per_step == m16.launches_per_step > 0
    assert not torch.equal(outs[0], outs[2]) or name == 'lm_mini'   # FP8 changes results on purpose


@pytest.mark.gpu
@pytest.mark.parametrize('name,pe', [('lm_mini', 'sin'), ('lm_mini', 'rope')])
def test_fp8_session_equals_generate_alone(monkeypatch, all_fp8, name, pe):
    """A request in a default (contiguous) session equals FP8 generate of it alone with ACB_LM_PREFILL=0."""
    from tests import test_gpu_continuous as TC
    TC.test_greedy_session_equals_generate_alone(monkeypatch, name, pe)


@pytest.mark.gpu
@pytest.mark.parametrize('slots', [4, 40])
def test_fp8_request_independent_of_neighbours(all_fp8, slots):
    from tests import test_gpu_continuous as TC
    TC.test_request_is_independent_of_slot_neighbours_and_history(slots, 'rope')


@pytest.mark.gpu
@pytest.mark.parametrize('slots', [4, 40])
def test_fp8_paged_session_equals_contiguous(all_fp8, slots):
    from tests import test_gpu_continuous_paged as TP
    TP.test_paged_session_equals_contiguous(slots, 'sin')


@pytest.mark.gpu
def test_fp8_prefilled_session_equals_generate_alone(monkeypatch, all_fp8):
    """A request in a prefill_prompts=True session equals FP8 generate on its default (prefilled) path."""
    from tests import test_gpu_continuous_prefill as TPF
    TPF.test_prefilled_session_equals_generate_alone(40, True, monkeypatch)


@pytest.mark.gpu
def test_fp8_weights_with_fp8_kv_requests_equal_alone(monkeypatch, all_fp8):
    """Paged sessions with kv_cache_dtype='fp8' on FP8 weights: each MusicGen request equals itself alone."""
    from tests import test_gpu_continuous_fp8kv as TF
    TF.test_fp8_musicgen_requests_equal_alone(monkeypatch)


@pytest.mark.gpu
def test_fp8_melody_continuous_equals_generate_with_chroma(monkeypatch, all_fp8):
    from tests import test_gpu_continuous_melody as TM
    TM.test_melody_continuous_equals_generate_alone(monkeypatch)


@pytest.mark.gpu
def test_fp8_stereo_melody_continuous_equals_generate(monkeypatch, all_fp8):
    from tests import test_gpu_continuous_melody as TM
    TM.test_stereo_melody_continuous_equals_generate_alone(monkeypatch)


@pytest.mark.gpu
def test_fp8_generate_stream_equals_generate(all_fp8):
    """The pieces of generate_stream, concatenated, equal generate: a melody model, and stereo over a long window."""
    from tests import test_gpu_streaming as TS
    TS.test_generate_stream_melody()
    TS.test_generate_stream_stereo_and_long_window()


@pytest.mark.gpu
def test_fp8_musicgen_text_continuous_equals_generate(monkeypatch, all_fp8):
    from tests import test_gpu_continuous as TC
    TC.test_musicgen_continuous_equals_generate(monkeypatch)


@pytest.mark.gpu
def test_fp8_stereo_generate_shape(all_fp8):
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/stereo-small', weight_dtype='fp8')
    assert mg.lm.weight_dtype == 'fp8'
    mg.set_generation_params(duration=0.5, top_k=50)
    torch.manual_seed(0)
    wav = mg.generate(['a', 'b'])
    assert wav.shape[:2] == (2, 2) and bool(torch.isfinite(wav).all())
