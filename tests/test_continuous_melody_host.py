"""Continuous batching of melody models on the host: the prefix bound a session is sized for, and the refusals raised before
any device work (a melody with a prompt, a melody on a model without a melody conditioner, a description longer than
max_text, a request without a prefix on a prefix model or with one on another model, a prefix longer than the session's)."""
import contextlib
import itertools
import types

import pytest
import torch

from audiocraft_b200.batching import ContinuousGenerator, Request, SlotSession, prefix_bound
from audiocraft_b200.conditioners import ConditionFuser


class _Stop(Exception):
    pass


def _no_device(*a, **k):
    raise AssertionError('device work before the refusal')


def _melody_lm(prepend=('self_wav', 'description'), chroma_len=235, match_len=True, cross=False):
    chroma = types.SimpleNamespace(chroma_len=chroma_len, match_len_on_eval=match_len)
    fuser = ConditionFuser({'prepend': list(prepend), **({'cross': ['description']} if cross else {})})
    return types.SimpleNamespace(has_prefix=True, cross_attention=cross, fuser=fuser, dim=8, n_q=4, card=16, cfg_coef=3.0,
                                 condition_provider=types.SimpleNamespace(conditioners={'self_wav': chroma}))


def test_prefix_bound():
    assert prefix_bound(types.SimpleNamespace(has_prefix=False), 64) == 0
    assert prefix_bound(_melody_lm(), 64) == 235 + 64          # [self_wav, description]: chroma + the longest description
    assert prefix_bound(_melody_lm(), 16) == 235 + 16
    assert prefix_bound(_melody_lm(('self_wav',), cross=True), 64) == 235   # [self_wav]: the chroma alone
    with pytest.raises(NotImplementedError):
        prefix_bound(_melody_lm(match_len=False), 64)          # the chroma follows the melody's length: no bound
    with pytest.raises(NotImplementedError):
        prefix_bound(types.SimpleNamespace(has_prefix=True, condition_provider=None), 64)


def test_session_sizes_the_cache_for_the_prefix(monkeypatch):
    """The KV cache holds max_prefix + the longest sequence (max_gen_len + max_delay + 1)."""
    from audiocraft_b200.patterns import DelayedPatternProvider
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    seen = {}

    def ensure(rows, seq_len, text_len, batch):
        seen.update(rows=rows, seq_len=seq_len, text_len=text_len, batch=batch)
        raise _Stop

    for lm, max_prefix, want in ((_melody_lm(), None, 235 + 32), (_melody_lm(), 100, 100),
                                 (_melody_lm(('self_wav',), cross=True), None, 235)):
        lm.pattern_provider = DelayedPatternProvider(4, delays=[0, 1, 2, 3])
        lm.special_token_id, lm.device, lm._ensure = 16, 'cpu', ensure
        with pytest.raises(_Stop):
            SlotSession(lm, 3, 50, max_text=32, max_prefix=max_prefix)
        assert seen['seq_len'] == want + 50 + 3 + 1 and seen['rows'] == 6 and seen['batch'] == 3
    text_lm = types.SimpleNamespace(has_prefix=False)
    with pytest.raises(ValueError, match='max_prefix'):
        SlotSession(text_lm, 2, 10, max_prefix=5)
    with pytest.raises(ValueError, match='max_prefix'):
        SlotSession(_melody_lm(), 2, 10, max_prefix=-1)


def _bare_session(lm, max_prefix=40):
    sess = SlotSession.__new__(SlotSession)
    lm._session = sess
    sess.lm, sess.max_gen_len, sess.max_prefix, sess.max_text = lm, 10, max_prefix, 8
    sess.sampling = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0)
    return sess


def test_admission_prefix_refusals(monkeypatch):
    monkeypatch.setattr('audiocraft_b200.batching.pattern_sequence', _no_device)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    lm = _melody_lm()
    lm.device = 'cpu'
    sess = _bare_session(lm)
    with pytest.raises(ValueError, match='needs its prefix'):
        sess.admit(0, Request(5))
    for bad in (torch.zeros(1, 4, 8), torch.zeros(2, 4, 7), torch.zeros(2, 4)):
        with pytest.raises(ValueError, match=r'prefix must be \[2, P'):
            sess.admit(0, Request(5, prefix=bad))
    with pytest.raises(ValueError, match='holds 0 .. 40'):
        sess.admit(0, Request(5, prefix=torch.zeros(2, 41, 8)))
    with pytest.raises(AssertionError, match='device work'):   # a prefix that fits gets as far as the sequence
        sess.admit(0, Request(5, prefix=torch.zeros(2, 40, 8)))
    sess = _bare_session(types.SimpleNamespace(has_prefix=False, dim=8))
    with pytest.raises(ValueError, match='must not carry one'):
        sess.admit(0, Request(5, prefix=torch.zeros(2, 3, 8)))


def _fake_model(melody=True):
    lm = _melody_lm() if melody else types.SimpleNamespace(has_prefix=False, cross_attention=True, n_q=4, card=16,
                                                            cfg_coef=3.0)
    gp = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0, two_step_cfg=False, cfg_coef_beta=None)
    return types.SimpleNamespace(lm=lm, generation_params=gp, max_duration=2.0, duration=1.0, frame_rate=50,
                                 sample_rate=32000, audio_channels=1, _has_melody=melody)


def _generator(model, max_prefix=235 + 8):
    gen = ContinuousGenerator.__new__(ContinuousGenerator)
    gen.model = model
    gen.defaults = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0)
    gen.session = types.SimpleNamespace(max_text=8, max_prefix=max_prefix)
    gen.scheduler = types.SimpleNamespace(submit=_no_device)
    gen._ids = itertools.count()
    return gen


def test_submit_melody_refusals_before_device_work():
    m = _fake_model()
    m._prepare_melody = m._prepare_tokens_and_attributes = _no_device
    gen = _generator(m)
    mel = torch.zeros(1, 3200)
    with pytest.raises(ValueError, match='prompt'):
        gen.submit('x', duration=1.0, melody=mel, melody_sample_rate=32000, prompt=torch.zeros(1, 100), prompt_sample_rate=32000)
    with pytest.raises(ValueError, match='melody_sample_rate'):
        gen.submit('x', duration=1.0, melody=mel)
    for bad in (torch.zeros(3200), torch.zeros(2, 1, 3200)):
        with pytest.raises(ValueError, match='one item'):
            gen.submit('x', duration=1.0, melody=bad, melody_sample_rate=32000)
    with pytest.raises(NotImplementedError, match='max_duration'):
        gen.submit('x', duration=5.0, melody=mel, melody_sample_rate=32000)
    for ok in (mel, mel[None]):   # [C, T] and [1, C, T] reach the chroma front-end
        with pytest.raises(AssertionError, match='device work'):
            gen.submit('x', duration=1.0, melody=ok, melody_sample_rate=32000)
    text = _fake_model(melody=False)
    text._prepare_tokens_and_attributes = _no_device
    with pytest.raises(NotImplementedError, match='melody'):
        _generator(text).submit('x', duration=1.0, melody=mel, melody_sample_rate=32000)


def test_submit_refuses_a_description_longer_than_max_text():
    m = _fake_model()
    m._prepare_tokens_and_attributes = lambda descriptions, prompt: ([descriptions], None)
    prefixes = {'short': torch.zeros(2, 235 + 3, 8), 'long': torch.zeros(2, 235 + 9, 8)}
    m.lm._condition_tensors = lambda attributes: (None, prefixes[attributes[0][0]])
    gen = _generator(m)
    with pytest.raises(ValueError, match='longer than 8 text positions'):
        gen.submit('long', duration=1.0)
    with pytest.raises(AssertionError, match='device work'):   # the short one is queued (the fake scheduler refuses it)
        gen.submit('short', duration=1.0)


def test_generator_takes_melody_models(monkeypatch):
    """The melody model's session is made with the prefix bound; a melody conditioner without a prefix, or a prefix without
    a melody conditioner, stays refused."""
    made = {}

    def session(self, lm, slots, max_gen_len, max_text, **kw):
        made.update(lm=lm, slots=slots, max_prefix=prefix_bound(lm, max_text))
        raise _Stop
    monkeypatch.setattr(SlotSession, '__init__', session)
    with pytest.raises(_Stop):
        ContinuousGenerator(_fake_model(), slots=3, max_text=16)
    assert made['max_prefix'] == 235 + 16 and made['slots'] == 3
    m = _fake_model()
    m.lm.has_prefix = False
    with pytest.raises(NotImplementedError, match='melody'):
        ContinuousGenerator(m)
