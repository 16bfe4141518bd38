"""FP8 LM weights on the host: the row quantizer against the float64 nearest-even search of the FP8 KV pool's tests, the
refusal of an unknown weight_dtype before any device work, and the C-ABI fields the format adds.

Format (include/audiocraft_b200.h, acb_lm_config.weight_dtype = 1): each output row n of a per-layer matrix has one fp32
scale, amax = max_k |W[n, k]|, code = e4m3(W * (448 / amax)) rounded to nearest even and saturated at +-448, scale =
amax / 448, both divisions correctly rounded; a zero row has zero codes and a zero scale."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from audiocraft_b200 import _lib, loaders
from audiocraft_b200 import lm as lm_mod
from audiocraft_b200.lm import E4M3_MAX, LMModel, quantize_rows_e4m3
from audiocraft_b200.musicgen import AudioGen, MusicGen
from tests.test_continuous_fp8kv_host import _e4m3_table, nearest_even64

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'audiocraft_b200.h')


def _check_rows(w, what):
    """quantize_rows_e4m3(w) against float64: every code the nearest-even e4m3 value of the fp32 product w * inv, every
    scale fp32(amax / 448) with the quotient taken in float64 (exact enough that its fp32 rounding is the correct one)."""
    codes, scales = quantize_rows_e4m3(w)
    assert codes.dtype == torch.float8_e4m3fn and codes.shape == w.shape and scales.shape == w.shape[:-1]
    x = w.float()
    amax = x.abs().amax(-1)
    live = amax > 0
    inv = torch.where(live, (E4M3_MAX / amax.double().clamp_min(1e-300)).float(), torch.zeros_like(amax))
    want = nearest_even64(x * inv.unsqueeze(-1))
    want = torch.where(live.unsqueeze(-1), want, torch.zeros_like(want))
    got = codes.double()
    bad = (got != want) | (torch.signbit(got) != torch.signbit(want)) & (want != 0)
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} codes differ from the float64 nearest-even search'
    sc_want = torch.where(live, (amax.double() / E4M3_MAX).float(), torch.zeros_like(amax))
    assert torch.equal(scales, sc_want), f'{what}: scales are not amax / 448 correctly rounded'
    assert not bool(codes[~live].view(torch.uint8).any()), f'{what}: a zero row has non-zero codes'
    return codes, scales


def test_row_quantizer_matches_nearest_even_search():
    g = torch.Generator().manual_seed(5)
    # random rows at the decode GEMMs' K (d and 4 d of MusicGen-medium), fp16 like the loaded weights, several magnitudes
    for K in (64, 1536, 6144):
        for sc in (2e-3, 0.05, 1.0, 300.0):
            _check_rows((torch.randn(24, K, generator=g) * sc).half(), f'random K={K} x{sc}')
    _check_rows(torch.rand(40, 1536, generator=g) * torch.logspace(-6, 3, 1536), 'fp32 rows over 9 decades')
    _check_rows((torch.randn(3, 7, 256, generator=g)).half(), 'stacked [..., K]')

    # ties: amax 448 (inv = 1 exactly) and every midpoint between two adjacent finite codes, of both signs
    _, vals = _e4m3_table()
    pos = torch.unique(vals[vals >= 0]).float()
    mids = ((pos[:-1].double() + pos[1:].double()) / 2).float()
    row = torch.cat([torch.tensor([448.0]), mids, -mids])
    codes, _ = _check_rows(row.unsqueeze(0), 'ties')
    y = torch.tensor([[448.0, 2.0 ** -10, 3 * 2.0 ** -10, 1.0625, 1.1875]])
    assert quantize_rows_e4m3(y)[0].float()[0].tolist() == [448.0, 0.0, 2.0 ** -8, 1.0, 1.25]

    # saturation: the amax element of each row codes to exactly +-448, also where x * (448 / amax) rounds above 448 in fp32
    x = torch.randn(2000, 64, generator=g) * 3
    prod = x.abs().amax(-1) * (E4M3_MAX / x.abs().amax(-1))
    assert bool((prod > E4M3_MAX).any()), 'some rows round their amax product above 448'
    codes, _ = _check_rows(x, 'saturation')
    j = x.abs().argmax(-1)
    hot = codes.float()[torch.arange(x.shape[0]), j]
    assert torch.equal(hot, torch.where(x[torch.arange(x.shape[0]), j] > 0, 448.0, -448.0))

    # zero rows (and -0) beside live rows: zero codes, zero scale
    x = torch.randn(4, 128, generator=g).half()
    x[1] = 0
    x[3] = -0.0
    codes, scales = _check_rows(x, 'zero rows')
    assert scales[1] == 0 and scales[3] == 0 and scales[0] > 0


class _DeviceWork(AssertionError):
    pass


def _no_device(*a, **k):
    raise _DeviceWork('device work before the refusal')


@pytest.mark.parametrize('bad', ['int8', 'FP8', 'bf16', None, 1])
def test_bad_weight_dtype_is_refused_before_device_work(monkeypatch, bad):
    monkeypatch.setattr(_lib, 'require_cuda', _no_device)
    monkeypatch.setattr(_lib, 'lib', _no_device)
    monkeypatch.setattr(loaders.synth, 'synth_lm_state_dict', _no_device)
    monkeypatch.setattr(loaders, 'load_compression_model', _no_device)
    with pytest.raises(ValueError, match='weight_dtype'):
        LMModel({}, {}, weight_dtype=bad)
    with pytest.raises(ValueError, match='weight_dtype'):
        loaders.load_lm_model('synthetic/small', device='cpu', weight_dtype=bad)
    with pytest.raises(ValueError, match='weight_dtype'):
        MusicGen.get_pretrained('synthetic/small', weight_dtype=bad)
    with pytest.raises(ValueError, match='weight_dtype'):
        AudioGen.get_pretrained('synthetic/audiogen-medium', weight_dtype=bad)
    for ok in ('fp16', 'fp8'):   # the accepted values get past the check (to the first device work)
        with pytest.raises(_DeviceWork):
            LMModel({}, {}, weight_dtype=ok)


def test_weight_dtype_codes():
    assert lm_mod.WEIGHT_DTYPES == {'fp16': 0, 'fp8': 1}


def _offsets_from_c(struct: str, fields):
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler to read the header layout')
    src = '#include <stddef.h>\n#include <stdio.h>\n#include "audiocraft_b200.h"\nint main(void) {\n'
    src += f'  printf("%zu\\n", sizeof({struct}));\n'
    src += ''.join(f'  printf("%zu\\n", offsetof({struct}, {f}));\n' for f in fields) + '  return 0;\n}\n'
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        c_path, exe = os.path.join(tmp, 'layout.c'), os.path.join(tmp, 'layout')
        with open(c_path, 'w') as fh:
            fh.write(src)
        subprocess.run([cc, '-I', os.path.dirname(HEADER), c_path, '-o', exe], check=True, capture_output=True)
        out = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    return out[0], out[1:]


def test_ctypes_layout_matches_the_header():
    fields = [f for f, _ in _lib.LMWeights._fields_]
    size, offs = _offsets_from_c('acb_lm_weights', fields)
    assert C.sizeof(_lib.LMWeights) == size
    assert [getattr(_lib.LMWeights, f).offset for f in fields] == offs
    assert fields[-7:] == ['s_qkv', 's_o', 's_cq', 's_ckv', 's_co', 's_ff1', 's_ff2'], 'the scales are appended'

    # acb_lm_config: the listed fields, then weight_dtype right after them in every instance, however it is built
    fields = [f for f, _ in _lib.LMConfig._fields_]
    size, offs = _offsets_from_c('acb_lm_config', fields + ['weight_dtype'])
    assert [getattr(_lib.LMConfig, f).offset for f in fields] == offs[:-1] and offs[-1] == C.sizeof(_lib.LMConfig)
    for cfg in (_lib.LMConfig(*range(12)), _lib.LMConfig(**{f: 3 for f in fields}), _lib.LMConfig(*range(12), weight_dtype=1)):
        assert C.sizeof(cfg) == size
        raw = C.c_int.from_address(C.addressof(cfg) + offs[-1]).value
        assert raw == cfg.weight_dtype in (0, 1)
    assert _lib.LMConfig(*range(12), weight_dtype=1).weight_dtype == 1 and _lib.LMConfig(*range(12)).weight_dtype == 0
