"""GPU: streaming generation.

* `acb_lstm_recurrent_carry` on each of its three kernels: a sequence run as ragged pieces with the state carried between calls
  is bit-identical to one call (y and the final state); from a zero state it is bit-identical to `acb_lstm_recurrent`; from a
  random state it stays within the float64 bound of the existing LSTM tests.
* `EncodecModel.stream_decoder` against `decode` on the tiny / tiny-causal / 24 kHz / 32 kHz codecs and the interleaved stereo
  wrapper, at 1, 8 and 33 items, pushed 1 frame, 7 frames, a seeded ragged schedule and one chunk at a time.
* `generate_stream` against the non-streaming call with the same seed: tokens equal, waveforms within 1e-5, and the first piece
  arrives before the last decode step.
"""
import os

import pytest
import torch

from audiocraft_b200 import synth
from tests import helpers as H

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-5


def _lib():
    from audiocraft_b200 import _lib as lib
    return lib, lib.lib()


# ----------------------------------------------------------------------------- LSTM recurrence with a carried state

def _lstm_run(L, lib, gx, w_hh, skip, B, Hd, h=None, c=None):
    T = gx.shape[-1]
    y = torch.empty((B, Hd, T), device='cuda')
    ws = torch.empty(int(L.acb_lstm_state_bytes(B, Hd)) // 4, device='cuda')
    if h is None:
        lib.check(L.acb_lstm_recurrent(lib.ptr(gx), lib.ptr(w_hh), lib.ptr(skip), lib.ptr(y), lib.ptr(ws), B, Hd, T,
                                       lib.stream()), 'lstm_recurrent')
    else:
        lib.check(L.acb_lstm_recurrent_carry(lib.ptr(gx), lib.ptr(w_hh), lib.ptr(skip), lib.ptr(y), lib.ptr(ws), lib.ptr(h),
                                             lib.ptr(c), B, Hd, T, lib.stream()), 'lstm_recurrent_carry')
    return y


def _lstm_f64(gx, w_hh, h, c):
    """nn.LSTM's recurrence in float64 from (h0, c0), gates_x given: [B, 4H, T] -> y [B, H, T], (h, c)."""
    gx, w_hh, h, c = gx.double().cpu(), w_hh.double().cpu(), h.double().cpu(), c.double().cpu()
    Hd, ys = h.shape[1], []
    for t in range(gx.shape[-1]):
        i, f, g, o = (gx[..., t] + h @ w_hh.t()).split(Hd, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        ys.append(h)
    return torch.stack(ys, dim=-1), h, c


@pytest.mark.parametrize('hidden,B', [(1024, 1), (1024, 8), (1024, 32),   # lstm_h2_kernel
                                      (192, 17),                             # lstm_tc_kernel (hidden % 64, not % 128)
                                      (1024, 33), (256, 33)])                # lstm_kernel (fp32 FMA, more than 32 items)
def test_lstm_carry_pieces_equal_one_call(hidden, B):
    lib, L = _lib()
    g = torch.Generator().manual_seed(hidden + B)
    T = 37
    gx = (torch.randn(B, 4 * hidden, T, generator=g) * 0.5).cuda()
    w_hh = (torch.randn(4 * hidden, hidden, generator=g) / hidden ** 0.5).cuda()
    skip = torch.randn(B, hidden, T, generator=g).cuda()
    h0 = (torch.rand(B, hidden, generator=g) * 2 - 1).cuda()
    c0 = torch.randn(B, hidden, generator=g).cuda()

    h, c = h0.clone(), c0.clone()
    whole = _lstm_run(L, lib, gx, w_hh, skip, B, hidden, h, c)
    hp, cp = h0.clone(), c0.clone()
    pieces = [_lstm_run(L, lib, gx[..., a:b].contiguous(), w_hh, skip[..., a:b].contiguous(), B, hidden, hp, cp)
              for a, b in ((0, 5), (5, 6), (6, T))]
    assert torch.equal(torch.cat(pieces, dim=-1), whole)
    assert torch.equal(hp, h) and torch.equal(cp, c)

    # from a zero state: the bits of acb_lstm_recurrent
    hz, cz = torch.zeros_like(h0), torch.zeros_like(c0)
    assert torch.equal(_lstm_run(L, lib, gx, w_hh, skip, B, hidden, hz, cz), _lstm_run(L, lib, gx, w_hh, skip, B, hidden))

    # against float64 from the random state, within the bound of the existing LSTM tests (rtol 1e-4, atol 2e-5)
    y64, h64, c64 = _lstm_f64(gx, w_hh, h0, c0)
    ref = y64 + skip.double().cpu()
    err = (whole.double().cpu() - ref).abs()
    assert (err <= 2e-5 + 1e-4 * ref.abs()).all(), f'max err {err.max():.2e}'
    assert ((h.double().cpu() - h64).abs() <= 2e-5 + 1e-4 * h64.abs()).all()
    assert ((c.double().cpu() - c64).abs() <= 2e-5 + 1e-4 * c64.abs()).all()
    print(f'lstm carry H={hidden} B={B}: max err vs float64 {err.max():.2e}')


# ----------------------------------------------------------------------------- stream decoder

def _schedules(n, seed):
    g = torch.Generator().manual_seed(seed)
    ragged, left = [], n
    while left > 0:
        k = min(left, int(torch.randint(0, 6, (1,), generator=g)))
        ragged.append(k)
        left -= k
    return {'1': [1] * n, '7': [7] * (n // 7) + ([n % 7] if n % 7 else []), 'ragged': ragged, 'one': [n]}


def _stream_decode(model, codes, schedule):
    dec = model.stream_decoder(codes.shape[0])
    out, t = [], 0
    for n in schedule:
        out.append(dec.push(codes[..., t:t + n]))
        t += n
    out.append(dec.flush())
    return torch.cat(out, dim=-1)


def _codes(cfg, name, B, T, seed):
    path = os.path.join(H.GOLDEN_DIR, f'{name}.pt')
    if B == 1 and os.path.exists(path):
        return torch.load(path, weights_only=False)['codes'][:1, :, :T].cuda()
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg['bins'], (B, cfg['n_q'], T), generator=g).cuda()


@pytest.mark.parametrize('B', [1, 8, 33])
@pytest.mark.parametrize('name', ['encodec_tiny', 'encodec_tiny_causal', 'encodec_24k', 'encodec_32k'])
def test_stream_decoder_equals_decode(name, B):
    from audiocraft_b200.encodec import EncodecModel
    cfg = synth.ENCODEC_CONFIGS[name]
    m = EncodecModel(synth.synth_encodec_state_dict(cfg, seed=1), cfg)
    codes = _codes(cfg, name, B, 30, seed=B)
    want = m.decode(codes)
    for key, sched in _schedules(codes.shape[-1], seed=B).items():
        got = _stream_decode(m, codes, sched)
        assert got.shape == want.shape, (key, got.shape, want.shape)
        err = (got - want).abs().max().item()
        print(f'{name} B={B} schedule {key}: max |stream - decode| {err:.2e}')
        assert err <= WAV_TOL, (key, err)


@pytest.mark.parametrize('B', [1, 8, 33])
def test_stereo_stream_decoder_equals_decode(B):
    from audiocraft_b200.encodec import EncodecModel, InterleaveStereoCompressionModel
    cfg = synth.ENCODEC_CONFIGS['encodec_32k']
    w = InterleaveStereoCompressionModel(EncodecModel(synth.synth_encodec_state_dict(cfg, seed=2), cfg))
    g = torch.Generator().manual_seed(B)
    codes = torch.randint(0, cfg['bins'], (B, 2 * cfg['n_q'], 23), generator=g).cuda()
    want = w.decode(codes)
    for key, sched in _schedules(codes.shape[-1], seed=B + 1).items():
        got = _stream_decode(w, codes, sched)
        assert got.shape == want.shape and got.shape[1] == 2
        err = (got - want).abs().max().item()
        print(f'stereo B={B} schedule {key}: max |stream - decode| {err:.2e}')
        assert err <= WAV_TOL, (key, err)


# ----------------------------------------------------------------------------- generate_stream

def _collect(mg, steps, **kw):
    """Runs generate_stream; returns (wav, tokens, progress count when the first non-empty piece arrived)."""
    wavs, toks, first_at = [], [], None
    for wav, tok in mg.generate_stream(return_tokens=True, progress=True, **kw):
        if wav.shape[-1] and first_at is None:
            first_at = steps[-1][0] if steps else 0
        wavs.append(wav)
        toks.append(tok)
    return torch.cat(wavs, dim=-1), torch.cat(toks, dim=-1), first_at


def _check(mg, call, stream_kw, seed=5, chunk=0.2):
    steps = []
    mg.set_custom_progress_callback(lambda done, total: steps.append((done, total)))
    torch.manual_seed(seed)
    wav, tok = call()
    steps.clear()
    torch.manual_seed(seed)
    swav, stok, first_at = _collect(mg, steps, chunk_duration=chunk, **stream_kw)
    mg.set_custom_progress_callback(None)
    assert torch.equal(stok, tok), 'streamed tokens differ'
    assert swav.shape == wav.shape, (swav.shape, wav.shape)
    err = (swav - wav).abs().max().item()
    print(f'{mg.name}: max |stream - generate| {err:.2e}, first piece after {first_at} of {steps[-1]}')
    assert err <= WAV_TOL
    assert first_at is not None and first_at < steps[-1][0], (first_at, steps[-1])   # steps counted through `progress`


@pytest.fixture(scope='module')
def small():
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/small')
    mg.set_generation_params(duration=1.0)
    return mg


def test_generate_stream_text(small):
    _check(small, lambda: small.generate(['a', 'b'], return_tokens=True), dict(descriptions=['a', 'b']))


def test_generate_stream_unconditional(small):
    _check(small, lambda: small.generate_unconditional(2, return_tokens=True), dict(num_samples=2))


def test_generate_stream_continuation(small):
    prompt = H.audio_input(dict(sample_rate=32000, channels=1), 2, 16000, 3)
    _check(small, lambda: small.generate_continuation(prompt, 32000, ['a', 'b'], return_tokens=True),
           dict(descriptions=['a', 'b'], prompt=prompt, prompt_sample_rate=32000))


def test_generate_stream_melody():
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/melody')
    mg.set_generation_params(duration=1.0)
    melody = H.audio_input(dict(sample_rate=32000, channels=1), 2, 32000, 7)
    _check(mg, lambda: mg.generate_with_chroma(['x', 'y'], melody, 32000, return_tokens=True),
           dict(descriptions=['x', 'y'], melody_wavs=melody, melody_sample_rate=32000))
    _check(mg, lambda: mg.generate(['x'], return_tokens=True), dict(descriptions=['x']))   # null melody


def test_generate_stream_stereo_and_long_window():
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/stereo-small')
    mg.set_generation_params(duration=1.0)
    _check(mg, lambda: mg.generate(['s'], return_tokens=True), dict(descriptions=['s']))
    mg.max_duration = 2.0
    mg.set_generation_params(duration=3.0, extend_stride=1.0)
    _check(mg, lambda: mg.generate(['long one'], return_tokens=True), dict(descriptions=['long one']), chunk=0.3)


def test_generate_stream_single_block(small):
    """A chunk longer than the generation: one block of steps, the audio in the last pieces, still equal."""
    torch.manual_seed(9)
    wav, tok = small.generate(['a'], return_tokens=True)
    torch.manual_seed(9)
    pieces = list(small.generate_stream(['a'], chunk_duration=5.0, return_tokens=True))
    assert torch.equal(torch.cat([t for _, t in pieces], dim=-1), tok)
    assert (torch.cat([w for w, _ in pieces], dim=-1) - wav).abs().max().item() <= WAV_TOL
