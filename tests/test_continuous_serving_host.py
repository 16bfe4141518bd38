"""Continuous batching as a service, on the host: per-request sampling options and `chunk_duration` refused before any device
work, cancellation in the scheduler against a fake device session, and the cohort streaming of `batching.CohortStream` on the
oracle's decoder layers (tests/test_streaming_host.py's backend, one item at a time): each request's pieces must be exactly
what the request streamed alone gives (splitting and shrinking cohorts changes no sample), and the oracle's decode of its
codes within the planner tolerance of tests/test_streaming_host.py (a convolution over a window rounds differently from one
over the whole sequence on the CPU)."""
import os
import types

import pytest
import torch

from audiocraft_b200 import _lib, synth
from audiocraft_b200.batching import (CohortStream, ContinuousGenerator, ContinuousScheduler, Request, SlotSession,
                                      pattern_sequence, SLOT_ACTIVE, SLOT_FINISHED, SLOT_INACTIVE)
from audiocraft_b200.patterns import DelayedPatternProvider
from audiocraft_b200.streaming import DecoderStream
from oracle import encodec_oracle as EO
from tests import helpers as H
from tests.test_streaming_host import OracleBackend


class FakeLM:
    def __init__(self, n_q=4, delays=(0, 1, 2, 3), card=16):
        self.n_q, self.card, self.special_token_id = n_q, card, card
        self.pattern_provider = DelayedPatternProvider(n_q, delays=list(delays))
        self.has_prefix = False


class FakeSession:
    """Device stand-in: every active slot advances one column per step and finishes after S - 1 steps.  A request's codes are
    drawn from its id; `frames` returns them as the device's sequence would once they are final."""

    def __init__(self, lm, slots):
        self.lm, self.log = lm, []
        self.state = [[0, SLOT_INACTIVE, 0] for _ in range(slots)]
        self.req = [None] * slots
        self.max_delay = max(lm.pattern_provider.delays)

    @staticmethod
    def codes(lm, req):
        return torch.randint(0, lm.card, (1, lm.n_q, req.max_gen_len), generator=torch.Generator().manual_seed(100 + req.id))

    def admit(self, slot, req):
        assert self.state[slot][1] != SLOT_ACTIVE
        S = pattern_sequence(self.lm, req.prompt, req.max_gen_len)[0].shape[-1]
        req.meta['S'] = S
        self.state[slot] = [0, SLOT_ACTIVE, S]
        self.req[slot] = req
        self.log.append(('admit', slot, req.id, {k: getattr(req, k) for k in ('use_sampling', 'temp', 'top_k', 'top_p',
                                                                               'cfg_coef')}))

    def retire(self, slot):
        assert self.state[slot][1] != SLOT_INACTIVE
        self.state[slot][1] = SLOT_INACTIVE
        self.log.append(('retire', slot))

    def steps(self, n):
        self.log.append(('steps', n))
        for st in self.state:
            for _ in range(n):
                if st[1] == SLOT_ACTIVE:
                    st[0] += 1
                    if st[0] == st[2] - 1:
                        st[1] = SLOT_FINISHED

    def status(self):
        return [(p, s) for p, s, _ in self.state]

    def collect(self, slot, req):
        return self.codes(self.lm, req)

    def frames(self, slots, t0, t1):
        out = []
        for s in slots:
            assert self.state[s][1] != SLOT_INACTIVE and t1 <= self.state[s][0] - self.max_delay, 'a frame read before final'
            out.append(self.codes(self.lm, self.req[s])[..., t0:t1])
        return torch.cat(out, dim=0)


# ----------------------------------------------------------------------------- refusals before device work

def _fake_model(**params):
    lm = types.SimpleNamespace(has_prefix=False, n_q=4, card=16, cfg_coef=3.0)
    gp = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0, two_step_cfg=False, cfg_coef_beta=None)
    gp.update(params)
    return types.SimpleNamespace(lm=lm, generation_params=gp, max_duration=2.0, duration=1.0, frame_rate=50,
                                 _has_melody=False)


def _no_device(*a, **k):
    raise AssertionError('device work before the refusal')


@pytest.mark.parametrize('bad', [dict(temperature=-0.5), dict(temperature=float('nan')), dict(temperature=float('inf')),
                                 dict(top_k=-1), dict(top_k=2.5), dict(top_p=-0.1), dict(top_p=1.5),
                                 dict(top_p=float('nan')), dict(cfg_coef=float('inf')), dict(cfg_coef=float('nan'))])
def test_sampling_options_refused_before_device_work(bad):
    gen = ContinuousGenerator.__new__(ContinuousGenerator)
    gen.model = _fake_model()
    gen.model._prepare_tokens_and_attributes = _no_device
    gen.defaults = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0)
    with pytest.raises(ValueError):
        gen.submit('x', duration=1.0, **bad)
    with pytest.raises(AssertionError, match='device work'):   # the same call with valid options gets as far as the conditions
        gen.submit('x', duration=1.0, temperature=0.7, top_k=0, top_p=1.0, cfg_coef=0.0, use_sampling=False)


def test_chunk_duration_refusals_before_device_work(monkeypatch):
    from audiocraft_b200.encodec import EncodecModel, HFEncodecCompressionModel
    monkeypatch.setattr(SlotSession, '__init__', _no_device)
    m = _fake_model()
    for bad in (0, -1.0):
        with pytest.raises(ValueError, match='chunk_duration'):
            ContinuousGenerator(m, chunk_duration=bad)
    gn = EncodecModel.__new__(EncodecModel)
    gn.cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'], norm='time_group_norm')
    hf = HFEncodecCompressionModel.__new__(HFEncodecCompressionModel)
    hf.cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'])
    for codec in (gn, hf, object()):
        m.compression_model = codec
        with pytest.raises(NotImplementedError):
            ContinuousGenerator(m, chunk_duration=0.5)
    m.compression_model = gn                               # without chunk_duration the codec is not asked for a stream decoder
    with pytest.raises(AssertionError, match='device work'):
        ContinuousGenerator(m)


def test_session_refuses_bad_options_before_device_work(monkeypatch):
    """SlotSession.admit checks a request's own options before it writes anything."""
    sess = SlotSession.__new__(SlotSession)
    sess.lm = types.SimpleNamespace(_session=sess, device='cpu')
    sess.max_gen_len = 10
    sess.sampling = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0)
    monkeypatch.setattr('audiocraft_b200.batching.pattern_sequence', _no_device)
    with pytest.raises(ValueError, match='top_p'):
        sess.admit(0, Request(5, top_p=2.0))


# ----------------------------------------------------------------------------- scheduler: cancellation, options

def test_cancel_waiting_active_finished_unknown():
    lm = FakeLM()
    dev = FakeSession(lm, 2)
    sch = ContinuousScheduler(dev, 2)
    for i, n in enumerate([10, 3, 6, 4, 5]):
        sch.submit(Request(n, id=i))
    assert sch.cancel(3)                                   # waiting: dropped, the others keep their order
    assert [r.id for r in sch.waiting] == [0, 1, 2, 4]
    done = sch.poll()                                      # 0 and 1 admitted; 1 retires after 6 steps
    assert [r.id for r, _ in done] == [1]
    assert not sch.cancel(1), 'a finished request cannot be cancelled'
    assert not sch.cancel(99) and not sch.cancel(3), 'unknown or already cancelled'
    assert sch.cancel(0)                                   # active: its slot is retired on the device ...
    assert ('retire', 0) in dev.log and 0 not in sch.active and dev.state[0][1] == SLOT_INACTIVE
    done = sch.poll()                                      # ... and takes the next waiting request at the next poll
    admits = [e[1:3] for e in dev.log if e[0] == 'admit']
    assert admits == [(0, 0), (1, 1), (0, 2), (1, 4)], admits
    order = [r.id for r, _ in done]
    while sch.pending:
        order += [r.id for r, _ in sch.poll()]
    assert order == [4, 2], order                          # 4 (5 frames) admitted with 2 (6 frames) finishes first
    assert all(st != SLOT_ACTIVE for _, st in dev.status())


def test_fifo_order_around_cancellations():
    lm = FakeLM()
    dev = FakeSession(lm, 1)
    sch = ContinuousScheduler(dev, 1)
    for i in range(6):
        sch.submit(Request(2, id=i))
    sch.poll()                                             # 0 runs to its end
    assert sch.cancel(2) and sch.cancel(4)
    while sch.pending:
        sch.poll()
    assert [e[2] for e in dev.log if e[0] == 'admit'] == [0, 1, 3, 5]


def test_request_options_reach_admit():
    lm = FakeLM()
    dev = FakeSession(lm, 2)
    sch = ContinuousScheduler(dev, 2)
    sch.submit(Request(4, id=0))
    sch.submit(Request(4, id=1, use_sampling=True, temp=0.7, top_k=5, top_p=0.0, cfg_coef=7.0))
    sch.submit(Request(4, id=2, top_p=0.9))
    while sch.pending:
        sch.poll()
    got = {e[2]: e[3] for e in dev.log if e[0] == 'admit'}
    assert got[0] == dict(use_sampling=None, temp=None, top_k=None, top_p=None, cfg_coef=None)
    assert got[1] == dict(use_sampling=True, temp=0.7, top_k=5, top_p=0.0, cfg_coef=7.0)
    assert got[2]['top_p'] == 0.9 and got[2]['temp'] is None


# ----------------------------------------------------------------------------- cohort streaming on the oracle's layers

class PerItemBackend(OracleBackend):
    """The oracle's layers run one item at a time, so that, like the codec kernels, an item's samples do not depend on the
    batch it is in (CPU convolutions and LSTMs over a batch may round differently from the same item alone)."""

    def conv(self, L, x):
        return torch.cat([super(PerItemBackend, self).conv(L, x[i:i + 1]) for i in range(x.shape[0])])

    def convtr(self, L, x, trim_left, t_out):
        return torch.cat([super(PerItemBackend, self).convtr(L, x[i:i + 1], trim_left, t_out) for i in range(x.shape[0])])

    def lstm(self, L, x, state):
        h, c = state['hc']
        ys = []
        for i in range(x.shape[0]):
            st = {'lstm': state['lstm'], 'hc': (h[:, i:i + 1], c[:, i:i + 1])}
            ys.append(super().lstm(L, x[i:i + 1], st))
            h, c = h.clone(), c.clone()
            h[:, i:i + 1], c[:, i:i + 1] = st['hc']
        state['hc'] = (h, c)
        return torch.cat(ys)

    def lstm_select(self, L, state, items):
        h, c = state['hc']
        return {'lstm': state['lstm'], 'hc': (h[:, items].clone(), c[:, items].clone())}


class OracleStreamDecoder:
    """The interface CohortStream uses (push / flush / select) over DecoderStream on the oracle's layers."""

    def __init__(self, cfg, sd, batch, stream=None):
        self.cfg, self.sd, self.batch = cfg, sd, batch
        self.oracle = EO.EncodecOracle(sd, cfg)
        self.stream = stream or DecoderStream(synth.encodec_layers(cfg)['decoder'], cfg, PerItemBackend(sd), batch)
        self.calls = 0

    def _out(self, y):
        return torch.empty((self.batch, 1, 0)) if y is None else y

    def push(self, codes):
        assert codes.shape[0] == self.batch
        return self._out(self.stream.push(self.oracle.decode_latent(codes)))

    def flush(self):
        return self._out(self.stream.flush())

    def select(self, items):
        return OracleStreamDecoder(self.cfg, self.sd, len(items), self.stream.select(items))


def _codec():
    cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'])
    g = torch.load(os.path.join(H.GOLDEN_DIR, 'encodec_tiny.pt'), weights_only=False)
    return cfg, synth.synth_encodec_state_dict(cfg, seed=g['wseed'])


def test_cohort_streaming_equals_decode_of_each_request():
    cfg, sd = _codec()
    lm = FakeLM(n_q=cfg['n_q'], card=cfg['bins'])
    dev = FakeSession(lm, 3)
    sch = ContinuousScheduler(dev, 3, poll_steps=3)
    made = []
    stream = CohortStream(sch, lambda n: made.append(n) or OracleStreamDecoder(cfg, sd, n), dev.max_delay)
    lens = {0: 12, 1: 12, 2: 20, 3: 7, 4: 9, 5: 14, 6: 5, 7: 11}
    submit_at = {0: [0, 1, 2], 2: [3, 4], 5: [5, 6, 7]}    # poll -> ids submitted before it
    cancelled, cancel_poll = 5, 10                         # request 5 (admitted at poll 8) is cancelled mid-decode
    pieces = {i: [] for i in lens}
    tokens = {i: [] for i in lens}
    finals, polls = {}, 0
    solo, solo_out = {}, {i: [] for i in lens}             # each request alone, fed the same frames: what it could emit
    with torch.no_grad():
        while polls == 0 or sch.pending or polls <= max(submit_at):
            for i in submit_at.get(polls, []):
                sch.submit(Request(lens[i], id=i))
            if polls == cancel_poll:
                assert tokens[cancelled] and cancelled in [r.id for r in sch.active.values()], 'not mid-decode'
                assert stream.cancel(cancelled)
                assert not stream.cancel(cancelled)
            events = stream.poll()
            for rid, piece, tok, final in events:
                assert rid != cancelled or polls < cancel_poll, 'an event after the cancel'
                assert rid not in finals, 'an event after the final one'
                pieces[rid].append(piece)
                tokens[rid].append(tok)
                if rid not in solo:
                    solo[rid] = OracleStreamDecoder(cfg, sd, 1)
                solo_out[rid].append(solo[rid].push(tok))
                if final:
                    solo_out[rid].append(solo[rid].flush())
                want_n = sum(p.shape[-1] for p in solo_out[rid]) - sum(p.shape[-1] for p in pieces[rid][:-1])
                assert piece.shape[-1] == want_n, ('a piece held back', rid, polls, piece.shape[-1], want_n)
                if final:
                    finals[rid] = polls
            # every decoding request had each of its final frames handed to the codec in this poll
            for slot, req in sch.active.items():
                n_tok = sum(t.shape[-1] for t in tokens[req.id])
                assert n_tok == max(0, sch.pos[slot] - dev.max_delay), (req.id, n_tok, sch.pos[slot])
            polls += 1
    assert sorted(finals) == [i for i in lens if i != cancelled]
    assert finals[0] == finals[1], 'two requests of one cohort and length finish together'
    assert len(made) >= 3 and max(made) == 3
    worst = 0.0
    for i in finals:
        codes = torch.cat(tokens[i], dim=-1)
        assert torch.equal(codes, FakeSession.codes(lm, Request(lens[i], id=i)))
        got = torch.cat(pieces[i], dim=-1)
        want = EO.seanet_decode(EO.EncodecOracle(sd, cfg).decode_latent(codes), sd, cfg)
        assert got.shape == want.shape, (i, got.shape, want.shape)
        assert torch.equal(got, torch.cat(solo_out[i], dim=-1)), f'request {i}: the cohort changed a sample'
        worst = max(worst, (got - want).abs().max().item())
    print(f'{len(finals)} streamed requests, max |pieces - decode| {worst:.2e}, {stream.codec_calls} codec calls in {polls} polls')
    assert worst <= 1e-5


def test_header_declares_the_serving_entry_points():
    from audiocraft_b200 import build
    with open(os.path.join(build.HERE, '..', 'include', 'audiocraft_b200.h')) as fh:
        text = fh.read()
    assert 'int acb_lm_retire(acb_lm_t* lm, int slot, void* stream);' in text and 'acb_lm_retire' in _lib.EXPORTS
    assert 'const acb_lm_sampling* sampling, void* stream);' in text[text.index('int acb_lm_admit('):]
    assert '#define ACB_LM_SLOT_STRIDE 8' in text and _lib.ACB_LM_SLOT_STRIDE == 8
    assert f'#define ACB_LM_SLOT_SAMPLING_STRIDE {_lib.ACB_LM_SLOT_SAMPLING_STRIDE}' in text
    fields = [f for f, _ in _lib.LMBuffers._fields_]
    assert fields[-3:] == ['slot_sampling', 'slot_state', 'slot_mask']
    assert 'int32_t* slot_sampling;' in text
