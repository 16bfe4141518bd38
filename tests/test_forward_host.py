"""CPU tests of the full-sequence forward's host side: the pattern tables compute_predictions uses against the reference's
own (tests/golden/lm_predictions.pt), the workspace arithmetic and shape checks of acb_lm_forward (pure host code, no
device is touched), and the MAGNeT stage guard."""
import ctypes as C
import os

import pytest
import torch

from tests import helpers as H
from audiocraft_b200.patterns import DelayedPatternProvider


def _golden():
    return torch.load(os.path.join(H.GOLDEN_DIR, 'lm_predictions.pt'), weights_only=False)


@pytest.mark.parametrize('key', [(4, 11, (0, 1, 2, 3)), (8, 9, (0, 0, 1, 1, 2, 2, 3, 3)), (3, 6, (0, 0, 2))])
def test_revert_pattern_logits_matches_reference_tables(key):
    K, T, delays = key
    p = DelayedPatternProvider(K, delays=list(delays)).get_pattern(T)
    for (valid, S), (idx, mask) in _golden()['tables'][key].items():
        B, card = 2, 3
        logits = torch.randn(B, card, K, S)
        vals, got_idx, got_mask = p.revert_pattern_logits(logits, float('nan'), keep_only_valid_steps=valid)
        assert torch.equal(got_idx, idx) and torch.equal(got_mask, mask), (valid, S)
        flat = torch.cat([logits.reshape(B, card, -1), torch.full((B, card, 1), float('nan'))], dim=-1)
        torch.testing.assert_close(vals, flat[:, :, idx.reshape(-1)].reshape(B, card, K, T), rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize('valid', [True, False])
def test_build_pattern_sequence_and_prediction_mask_match_reference(valid):
    """The sequence compute_predictions builds has the reference's length, and the NaN pattern / mask of its predictions
    follow from the tables alone."""
    g = _golden()
    for name, case in g['cases'].items():
        from audiocraft_b200 import synth
        cfg = synth.lm_config(name)
        K, T = cfg['n_q'], case['T']
        p = DelayedPatternProvider(K, delays=cfg['delays']).get_pattern(T)
        codes = torch.randint(0, cfg['card'], (1, K, T))
        seq, _, smask = p.build_pattern_sequence(codes, cfg['card'], keep_only_valid_steps=valid)
        assert seq.shape[-1] == (T + 1 if valid else T + max(cfg['delays']) + 1)
        key = 'valid' if valid else 'all'
        _, mask = p.logits_tables(seq.shape[-1], valid)
        assert torch.equal(torch.from_numpy(mask), case[f'mask_{key}'])
        assert torch.equal(~torch.from_numpy(mask)[None].expand(case['batch'], -1, -1), case[f'nan_{key}'])


def _cfg(**over):
    from audiocraft_b200 import _lib
    f = dict(dim=256, num_heads=4, num_layers=3, ffn_dim=1024, n_q=4, card=128, cross_attention=1, max_rows=1, max_seq=2,
             max_text=1, pos_scale=1.0, positional_embedding=0)
    f.update(over)
    return _lib.LMConfig(*[f[n] for n, _ in _lib.LMConfig._fields_])


def _ws(cfg, B, P, S, Tt):
    from audiocraft_b200 import _lib, build
    build.build()
    return _lib.lib().acb_lm_forward_workspace_bytes(C.byref(cfg), B, P, S, Tt)


def test_forward_workspace_arithmetic():
    def up(n):
        return (n + 255) // 256 * 256
    B, P, S, Tt, d, ffn = 3, 5, 41, 7, 256, 1024
    M = B * (P + S)
    want = up(M * d * 4) + 5 * up(M * d * 2) + up(M * ffn * 2) + 3 * up(B * Tt * d * 2)
    assert _ws(_cfg(), B, P, S, Tt) == want
    # without cross attention the condition buffers take nothing, whatever text_len says
    assert _ws(_cfg(cross_attention=0), B, P, S, 0) == want - 3 * up(B * Tt * d * 2)
    # MusicGen-medium, 8 items x 1501 positions: the size the docs quote
    med = _ws(_cfg(dim=1536, num_heads=24, num_layers=48, ffn_dim=6144, card=2048), 8, 0, 1501, 16)
    assert 0.35e9 < med < 0.45e9
    # the largest shapes the launch grids take are accepted
    assert _ws(_cfg(), 65535, 0, 128, 1) > 0 and _ws(_cfg(), 1000, 0, 4, 8388) > 0


@pytest.mark.parametrize('over,args', [
    (dict(num_heads=3), (1, 0, 4, 1)),            # head_dim != 64
    (dict(dim=4096, num_heads=64), (1, 0, 4, 1)),  # dim above the LayerNorm kernel
    (dict(ffn_dim=1020), (1, 0, 4, 1)),           # ffn_dim not a multiple of 8
    (dict(card=127), (1, 0, 4, 1)),               # odd card
    (dict(n_q=17), (1, 0, 4, 1)),
    (dict(positional_embedding=3), (1, 0, 4, 1)),
    (dict(), (0, 0, 4, 1)),                       # empty batch
    (dict(), (1, 0, 0, 1)),                       # empty sequence
    (dict(), (1, -1, 4, 1)),                      # negative prefix
    (dict(), (1, 0, 4, 0)),                       # cross attention without text
    (dict(), (65535, 0, 129, 1)),                 # token rows beyond the GEMM grid (65535 tiles of 128 rows)
    (dict(), (1000, 0, 4, 8389)),                 # condition rows beyond it
    (dict(), (65536, 0, 1, 1)),                   # items beyond the attention grid
])
def test_forward_rejects_bad_shapes_without_a_device(over, args):
    from audiocraft_b200 import _lib, build
    build.build()
    L = _lib.lib()
    cfg = _cfg(**over)
    assert L.acb_lm_forward_workspace_bytes(C.byref(cfg), *args) == -1
    w = _lib.LMWeights(*([1] * len(_lib.LMWeights._fields_)))   # never dereferenced: the shape check comes first
    rc = L.acb_lm_forward(C.byref(cfg), C.byref(w), 1, 1, None, *args, 1, 1, 1 << 40, None)
    assert rc == -1 and L.acb_last_error()


def test_forward_rejects_small_workspace_and_missing_inputs():
    from audiocraft_b200 import _lib, build
    build.build()
    L = _lib.lib()
    cfg = _cfg()
    need = L.acb_lm_forward_workspace_bytes(C.byref(cfg), 2, 0, 9, 3)
    w = _lib.LMWeights(*([1] * len(_lib.LMWeights._fields_)))
    assert L.acb_lm_forward(C.byref(cfg), C.byref(w), 1, 1, None, 2, 0, 9, 3, 1, 1, need - 1, None) == -1
    assert b'workspace' in L.acb_last_error()
    assert L.acb_lm_forward(C.byref(cfg), C.byref(w), 1, None, None, 2, 0, 9, 3, 1, 1, need, None) == -1   # no condition
    assert L.acb_lm_forward(C.byref(cfg), C.byref(w), 1, 1, None, 2, 4, 9, 3, 1, 1, 1 << 40, None) == -1   # P without prefix


def test_stage_raises_without_a_device():
    from audiocraft_b200.lm import LMModel
    m = LMModel.__new__(LMModel)   # the guard comes before any device work
    with pytest.raises(NotImplementedError):
        m.forward(torch.zeros(1, 4, 3, dtype=torch.long), stage=0)
    with pytest.raises(NotImplementedError):
        m.compute_predictions(torch.zeros(1, 4, 3, dtype=torch.long), stage=1)
