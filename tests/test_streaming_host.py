"""CPU: the streaming decoder's planner (audiocraft_b200/streaming.py) driven by the oracle's layers, and the refusals of the
streaming API that need no device.

The planner only slices and joins; here its four layer operations are plain fp32 torch (F.conv1d, F.conv_transpose1d, nn.LSTM
given (h0, c0)), so a piece-by-piece decode must give `seanet_decode` of the whole latent to rounding.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from audiocraft_b200 import synth
from audiocraft_b200.streaming import DecoderStream
from oracle import encodec_oracle as EO
from tests import helpers as H


class OracleBackend:
    def __init__(self, sd):
        self.sd = sd

    def conv(self, L, x):
        w, b = EO._conv_weight(self.sd, L['prefix'])
        return F.conv1d(EO.elu(x) if L['elu'] else x, w, b, stride=L['stride'], dilation=L['dilation'])

    def resblock(self, block, x, pad_left):
        shortcut, a, b = block
        y = self.conv(b, self.conv(a, x))
        skip = x[..., pad_left:pad_left + y.shape[-1]]
        return (skip if shortcut is None else self.conv(shortcut, skip)) + y

    def convtr(self, L, x, trim_left, t_out):
        w, b = EO._conv_weight(self.sd, L['prefix'])
        y = F.conv_transpose1d(EO.elu(x) if L['elu'] else x, w, b, stride=L['stride'])
        return y[..., trim_left:trim_left + t_out]

    def lstm_state(self, L, batch):
        H_ = L['dim']
        lstm = torch.nn.LSTM(H_, H_, L['layers'])
        with torch.no_grad():
            for n in range(L['layers']):
                for k in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'):
                    getattr(lstm, f'{k}_l{n}').copy_(self.sd[f"{L['prefix']}{k}_l{n}"].float())
        return {'lstm': lstm, 'hc': (torch.zeros(L['layers'], batch, H_), torch.zeros(L['layers'], batch, H_))}

    def lstm(self, L, x, state):
        with torch.no_grad():
            y, state['hc'] = state['lstm'](x.permute(2, 0, 1), state['hc'])
        return y.permute(1, 2, 0) + x


def _schedules(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    ragged, left = [], n
    while left > 0:
        k = min(left, int(torch.randint(0, 6, (1,), generator=g)))   # 0-frame pushes included
        ragged.append(k)
        left -= k
    return {'1': [1] * n, '7': [7] * (n // 7) + ([n % 7] if n % 7 else []), 'ragged': ragged, 'one': [n]}


def _setup(name, cfg_over=None):
    cfg = dict(synth.ENCODEC_CONFIGS[name], **(cfg_over or {}))
    g = torch.load(os.path.join(H.GOLDEN_DIR, f'{name}.pt'), weights_only=False)
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    o = EO.EncodecOracle(sd, cfg)
    return cfg, sd, o, g['codes']


def _stream(cfg, sd, z, schedule):
    s = DecoderStream(synth.encodec_layers(cfg)['decoder'], cfg, OracleBackend(sd), z.shape[0])
    pieces, t = [], 0
    for n in schedule:
        pieces.append(s.push(z[..., t:t + n]))
        t += n
    pieces.append(s.flush())
    return torch.cat([p for p in pieces if p is not None], dim=-1), s


@pytest.mark.parametrize('pad_mode', ['reflect', 'constant'])
@pytest.mark.parametrize('name', ['encodec_tiny', 'encodec_tiny_causal', 'encodec_24k'])
def test_planner_reproduces_seanet_decode(name, pad_mode):
    cfg, sd, o, codes = _setup(name, {'pad_mode': pad_mode})
    z = o.decode_latent(codes)
    if name == 'encodec_24k':
        z = z[..., :40]
    with torch.no_grad():
        want = EO.seanet_decode(z, sd, cfg)
        for key, sched in _schedules(z.shape[-1], seed=z.shape[-1]).items():
            got, _ = _stream(cfg, sd, z, sched)
            assert got.shape == want.shape, (key, got.shape, want.shape)
            err = (got - want).abs().max().item()
            assert err <= 1e-5, (key, err)


@pytest.mark.parametrize('n', [1, 2, 3, 5])
def test_planner_short_sequences(n):
    """Latents shorter than a reflect pad: the layers that never started pad their whole input at flush, as pad1d does."""
    cfg, sd, o, codes = _setup('encodec_tiny')
    z = o.decode_latent(codes)[..., :n]
    with torch.no_grad():
        want = EO.seanet_decode(z, sd, cfg)
        got, _ = _stream(cfg, sd, z, [1] * n)
    assert got.shape == want.shape and (got - want).abs().max().item() <= 1e-5


@pytest.mark.parametrize('name', ['encodec_tiny', 'encodec_tiny_causal'])
def test_lookahead_matches_brute_force(name):
    """Perturb one frame at a time and record which output samples change.  The lookahead is the largest (changed frame -
    the sample's own frame) over samples past the start (a reflect pad's first window reaches further)."""
    cfg, sd, o, codes = _setup(name)
    z = o.decode_latent(codes)[:1]
    T = z.shape[-1]
    hop = int(torch.tensor(cfg['ratios']).prod())
    s = DecoderStream(synth.encodec_layers(cfg)['decoder'], cfg, OracleBackend(sd), 1)
    with torch.no_grad():
        base = EO.seanet_decode(z, sd, cfg)
        last = torch.full((base.shape[-1],), -1)
        for f in range(T):
            zp = z.clone()
            zp[..., f] += 1.0
            changed = ((EO.seanet_decode(zp, sd, cfg) - base).abs().amax(dim=(0, 1)) > 0)
            last[changed] = f
    o_idx = torch.arange(base.shape[-1])
    start = 8 * hop                        # past every layer's first window
    right = (last - o_idx // hop)[start:T * hop]
    assert int(right.max()) == s.lookahead, (int(right.max()), s.lookahead)


def test_streamed_pieces_are_final_after_lookahead():
    """After pushing n frames, every sample of frames < n - lookahead has been returned."""
    cfg, sd, o, codes = _setup('encodec_tiny')
    z = o.decode_latent(codes)[:1]
    hop = int(torch.tensor(cfg['ratios']).prod())
    s = DecoderStream(synth.encodec_layers(cfg)['decoder'], cfg, OracleBackend(sd), 1)
    got = 0
    with torch.no_grad():
        for n in range(1, z.shape[-1] + 1):
            y = s.push(z[..., n - 1:n])
            got += 0 if y is None else y.shape[-1]
            if n > 8:
                assert got >= (n - s.lookahead) * hop, (n, got)


def test_stream_decoder_refusals_before_device_work():
    """GroupNorm codecs and transformers' chunked codec refuse streaming; a renormalisation scale is refused.  All raise before
    any device work, so they run here (the model objects are built without __init__)."""
    from audiocraft_b200.encodec import EncodecModel, HFEncodecCompressionModel
    m = EncodecModel.__new__(EncodecModel)
    m.cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'], norm='time_group_norm')
    with pytest.raises(NotImplementedError, match='GroupNorm'):
        m.stream_decoder(1)
    m.cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'])
    with pytest.raises(NotImplementedError, match='scale'):
        m.stream_decoder(1, scale=torch.ones(1, 1))
    hf = HFEncodecCompressionModel.__new__(HFEncodecCompressionModel)
    hf.cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'])
    with pytest.raises(NotImplementedError):
        hf.stream_decoder(1)


def test_generate_stream_refusals_before_device_work():
    from audiocraft_b200.musicgen import MusicGen
    from audiocraft_b200.encodec import HFEncodecCompressionModel
    mg = MusicGen.__new__(MusicGen)
    for bad in (0, -1.0):
        with pytest.raises(ValueError):
            next(mg.generate_stream(['x'], chunk_duration=bad))
    mg.compression_model = HFEncodecCompressionModel.__new__(HFEncodecCompressionModel)
    mg.compression_model.cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'])
    with pytest.raises(NotImplementedError):
        next(mg.generate_stream(['x'], chunk_duration=1.0))
