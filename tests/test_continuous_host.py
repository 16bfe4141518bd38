"""Continuous batching on the host: the scheduler's FIFO admission and retirement against a fake device session, the
per-request sequence and mask against `LMModel._generate_begin`'s construction, and the refusals raised before any device
work."""
import types

import pytest
import torch

from audiocraft_b200 import _lib
from audiocraft_b200.batching import (ContinuousGenerator, ContinuousScheduler, Request, SlotSession, pattern_sequence,
                                      revert_sequence, SLOT_ACTIVE, SLOT_FINISHED)
from audiocraft_b200.patterns import DelayedPatternProvider


class FakeLM:
    def __init__(self, n_q=4, delays=(0, 1, 2, 3), card=16):
        self.n_q, self.card, self.special_token_id = n_q, card, card
        self.pattern_provider = DelayedPatternProvider(n_q, delays=list(delays))
        self.has_prefix = False


class FakeSession:
    """Device stand-in: every active slot advances one column per step and finishes after S - 1 steps; codes are the id."""

    def __init__(self, lm, slots):
        self.lm, self.state, self.log = lm, [[0, 0, 0] for _ in range(slots)], []

    def admit(self, slot, req):
        assert self.state[slot][1] != SLOT_ACTIVE
        S = pattern_sequence(self.lm, req.prompt, req.max_gen_len)[0].shape[-1]
        req.meta['S'] = S
        self.state[slot] = [0, SLOT_ACTIVE, S]
        self.log.append(('admit', slot, req.id))

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
        return torch.full((1, self.lm.n_q, req.max_gen_len), req.id)


def test_scheduler_fifo_admission_and_retirement():
    lm = FakeLM()
    dev = FakeSession(lm, 2)
    sch = ContinuousScheduler(dev, 2)
    lens = [10, 3, 5, 7, 2]
    for i, n in enumerate(lens):
        sch.submit(Request(n, id=i))
    order, polls = [], 0
    while sch.pending:
        order += [r.id for r, codes in sch.poll()]
        polls += 1
    admits = [(e[1], e[2]) for e in dev.log if e[0] == 'admit']
    assert admits[:2] == [(0, 0), (1, 1)], admits
    assert [a[1] for a in admits] == [0, 1, 2, 3, 4], 'FIFO admission'
    # steps: 1 retires at 6, 0 at 13, 2 (admitted at 6) at 14, 4 (admitted at 14) at 19, 3 (admitted at 13) at 23
    assert order == [1, 0, 2, 4, 3], order
    steps = sum(e[1] for e in dev.log if e[0] == 'steps')
    busy = sum(n + 3 for n in lens)                        # S - 1 = max_gen_len + max_delay steps each
    assert sch.steps_run == steps and sch.busy_slot_steps == busy
    assert 0 < sch.occupancy <= 1


def test_scheduler_poll_steps_and_device_mismatch():
    lm = FakeLM()
    dev = FakeSession(lm, 1)
    sch = ContinuousScheduler(dev, 1, poll_steps=4)
    sch.submit(Request(6, id=0))
    got = []
    while sch.pending:
        got += sch.poll()
    assert [e[1] for e in dev.log if e[0] == 'steps'] == [4, 4, 1]
    assert torch.equal(got[0][1], torch.zeros(1, 4, 6, dtype=torch.long))
    dev2 = FakeSession(lm, 1)
    dev2.steps = lambda n: None                            # a device that does not advance is caught at the next poll
    sch = ContinuousScheduler(dev2, 1)
    sch.submit(Request(3, id=0))
    with pytest.raises(RuntimeError, match='expected'):
        sch.poll()
    with pytest.raises(ValueError):
        ContinuousScheduler(dev, 1, poll_steps=0)


@pytest.mark.parametrize('n_q,delays', [(4, (0, 1, 2, 3)), (8, (0, 0, 1, 1, 2, 2, 3, 3))])
@pytest.mark.parametrize('T,T0', [(2, 0), (9, 0), (9, 4), (30, 29)])
def test_request_sequence_matches_generate_begin(n_q, delays, T, T0):
    lm = FakeLM(n_q, delays)
    prompt = torch.randint(0, lm.card, (1, n_q, T0)) if T0 else None
    seq, mask, pattern = pattern_sequence(lm, prompt, T)
    # _generate_begin's construction for a batch of one
    p = lm.pattern_provider.get_pattern(T)
    codes = torch.full((1, n_q, T), -1, dtype=torch.long)
    if T0:
        codes[..., :T0] = prompt
    want, _, want_mask = p.build_pattern_sequence(codes, lm.special_token_id)
    assert torch.equal(seq, want) and torch.equal(mask, want_mask)
    assert seq.shape[-1] == T + max(delays) + 1
    # a finished sequence reverts to the codes, prompt included
    full = torch.randint(0, lm.card, (1, n_q, T))
    if T0:
        full[..., :T0] = prompt
    done, _, _ = p.build_pattern_sequence(full, lm.special_token_id)
    assert torch.equal(revert_sequence(lm, done, mask, pattern, T), full)
    with pytest.raises(AssertionError):
        revert_sequence(lm, seq, mask, pattern, T)         # unknown tokens left: refused like _generate_end


def _fake_model(**params):
    lm = types.SimpleNamespace(has_prefix=False, n_q=4, card=16)
    gp = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0, two_step_cfg=False, cfg_coef_beta=None)
    gp.update(params)
    return types.SimpleNamespace(lm=lm, generation_params=gp, max_duration=2.0, duration=1.0, frame_rate=50,
                                 _has_melody=False)


def test_refusals_before_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError('device work before the refusal')
    monkeypatch.setattr(SlotSession, '__init__', no_device)
    with pytest.raises(NotImplementedError, match='two_step_cfg'):
        ContinuousGenerator(_fake_model(two_step_cfg=True))
    with pytest.raises(NotImplementedError, match='cfg_coef_beta'):
        ContinuousGenerator(_fake_model(cfg_coef_beta=2.0))
    m = _fake_model()
    m._has_melody = True
    with pytest.raises(NotImplementedError, match='melody'):
        ContinuousGenerator(m)
    m = _fake_model()
    m.lm.has_prefix = True
    with pytest.raises(NotImplementedError, match='prefix'):
        ContinuousGenerator(m)
    # duration beyond max_duration: refused at submit, before the conditions or the codec run
    gen = ContinuousGenerator.__new__(ContinuousGenerator)
    gen.model = _fake_model()
    gen.model._prepare_tokens_and_attributes = no_device
    with pytest.raises(NotImplementedError, match='max_duration'):
        gen.submit('x', duration=2.5)
    with pytest.raises(ValueError):
        gen.submit('x', duration=0.001)
    with pytest.raises(ValueError, match='prompt_sample_rate'):
        gen.submit('x', duration=1.0, prompt=torch.zeros(1, 100))


def test_session_argument_validation(monkeypatch):
    lm = types.SimpleNamespace(has_prefix=False)
    for slots in (0, _lib.ACB_LM_MAX_SLOTS + 1):
        with pytest.raises(ValueError):
            SlotSession(lm, slots, 10)
    with pytest.raises(ValueError):
        SlotSession(lm, 2, 0)
    lm.has_prefix = True
    with pytest.raises(NotImplementedError):
        SlotSession(lm, 2, 10)


def test_header_declares_the_slot_entry_points():
    import os
    from audiocraft_b200 import build
    with open(os.path.join(build.HERE, '..', 'include', 'audiocraft_b200.h')) as fh:
        text = fh.read()
    for name in ('acb_lm_begin_slots', 'acb_lm_admit', 'acb_lm_slot_status'):
        assert f'int {name}(' in text and name in _lib.EXPORTS
    assert '#define ACB_LM_SLOT_STRIDE 8' in text and _lib.ACB_LM_SLOT_STRIDE == 8
    fields = [f for f, _ in _lib.LMBuffers._fields_]
    assert fields[-2:] == ['slot_state', 'slot_mask']
