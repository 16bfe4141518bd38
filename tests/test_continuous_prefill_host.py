"""Prefilled prompts and window extension in continuous batching, on the host.

* `musicgen.window_plan` is the window loop of `BaseGenModel._token_windows` (driven by a fake window callable), over
  durations, max_duration / extend_stride pairs (MusicGen 30 / 18, AudioGen 10 / 2, a short test window), prompt lengths
  and frame rates; `batching.WindowChain` fed the same windows returns the same tokens.
* `ContinuousScheduler` against fake sessions: a slot starts at its prefilled column; a long request's next window is
  re-admitted in the poll its previous window finished, into the same slot and ahead of the waiting requests; in a tight
  page pool it takes the pages it released and no waiting request overtakes another; cancellation before, during and
  between windows; `CohortStream` frame accounting with members admitted together at different start columns.
* `ContinuousGenerator.submit` draws one seed per window, in `generate`'s order (each window's conditions, then its seed).
* Refusals before device work: extension with chunk_duration, and any duration past max_duration without prefill_prompts.
"""
import itertools
import types

import pytest
import torch

from audiocraft_b200.batching import (SLOT_ACTIVE, CohortStream, ContinuousGenerator, ContinuousScheduler, PagePool,
                                      Request, WindowChain, pattern_sequence, prefill_columns)
from audiocraft_b200.musicgen import BaseGenModel, window_plan
from tests.test_continuous_paged_host import FakePagedSession
from tests.test_continuous_serving_host import FakeLM, FakeSession


def _no_device(*a, **k):
    raise AssertionError('device work before the refusal')


# ----------------------------------------------------------------------------- the window plan

class FakeWindows:
    """A window callable for `_token_windows`: window k returns its prompt followed by frames drawn from seed k."""

    def __init__(self, K=4):
        self.K, self.calls = K, []

    def codes(self, k, prompt, n):
        T0 = 0 if prompt is None else prompt.shape[-1]
        assert T0 < n or (prompt is None and n > 0), (T0, n)
        new = torch.randint(0, 2048, (1, self.K, n - T0), generator=torch.Generator().manual_seed(k))
        return new if prompt is None else torch.cat([prompt, new], dim=-1)

    def __call__(self, prompt, attrs, n, callback):
        self.calls.append((0 if prompt is None else prompt.shape[-1], n, attrs))
        yield self.codes(len(self.calls) - 1, prompt, n)


def _genmodel(duration, max_duration, stride, fr):
    m = BaseGenModel.__new__(BaseGenModel)
    m.duration, m.max_duration, m.extend_stride, m._progress_callback = duration, max_duration, stride, None
    m.compression_model = types.SimpleNamespace(frame_rate=fr)
    m._window_attributes = lambda attrs, offset: ('attrs', offset)
    return m


WINDOWS = [(30.0, 18.0), (10.0, 2.0), (1.0, 0.4)]


@pytest.mark.parametrize('max_duration,stride', WINDOWS)
@pytest.mark.parametrize('fr', [50, 25, 12.5])
def test_window_plan_is_token_windows(max_duration, stride, fr):
    cases = 0
    for f in (0.25, 1.0, 1.02, 1.3, 2.5, 4.17):
        duration = round(max_duration * f, 3)
        n_total = int(duration * fr)
        first = int(min(duration, max_duration) * fr)
        for T0 in sorted({0, 1, 7, first // 2, first - 1}):
            if T0 >= first or n_total < 1:
                continue
            prompt = None if T0 == 0 else torch.randint(0, 2048, (1, 4, T0), generator=torch.Generator().manual_seed(T0))
            windows = FakeWindows()
            m = _genmodel(duration, max_duration, stride, fr)
            want = torch.cat(list(m._token_windows([], prompt, False, windows)), dim=-1)
            plan = window_plan(duration, max_duration, stride, fr, T0)
            assert [(w.prompt_len, w.length) for w in plan] == [c[:2] for c in windows.calls]
            if duration > max_duration:
                assert [('attrs', w.time_offset) for w in plan] == [c[2] for c in windows.calls]
                assert [w.start for w in plan] == [k * int(fr * stride) for k in range(len(plan))]
                assert all(w.time_offset == w.start / fr for w in plan)
                assert all(w.length <= plan[0].length for w in plan), 'a later window is longer than the first'
            # the session's chain over the same windows gives the same tokens
            made = []
            chain = WindowChain(plan, lambda k, p: made.append((k, p)) or Request(plan[k].length, prompt=p, id=k),
                                prompt if duration > max_duration else None)
            if duration <= max_duration:
                assert len(plan) == 1 and torch.equal(FakeWindows().codes(0, prompt, plan[0].length), want)
                continue
            req, k = chain.make(0, prompt), 0
            while req is not None:
                req = chain.advance(FakeWindows().codes(k, req.prompt, req.max_gen_len))
                k += 1
            assert k == len(plan) and [i for i, _ in made] == list(range(len(plan)))
            assert torch.equal(chain.tokens(), want)
            cases += 1
    assert cases >= 4


def test_window_plan_refusals():
    with pytest.raises(AssertionError, match='Stride should be defined'):
        window_plan(31, 30, None, 50)
    with pytest.raises(AssertionError, match='Cannot stride'):
        window_plan(31, 30, 30, 50)
    assert len(window_plan(30, 30, None, 50, 10)) == 1


# ----------------------------------------------------------------------------- scheduler and stream

class PrefillSession(FakeSession):
    """FakeSession whose slot starts at the request's prefilled column; a request's codes keep its prompt."""

    def admit(self, slot, req):
        super().admit(slot, req)
        self.state[slot][0] = req.prefill_cols

    def positions(self, req):
        return pattern_sequence(self.lm, None, req.max_gen_len)[0].shape[-1]

    @staticmethod
    def codes(lm, req):
        c = FakeSession.codes(lm, req)
        if req.prompt is not None:
            c[..., :req.prompt.shape[-1]] = req.prompt
        return c


class PagedPrefillSession(FakePagedSession):
    def admit(self, slot, req):
        super().admit(slot, req)
        self.state[slot][0] = req.prefill_cols
        self.log.append(('pages', slot, req.id, list(self.pages.held[slot])))

    codes = staticmethod(PrefillSession.codes)


def _prompt(lm, T0, seed):
    return torch.randint(0, lm.card, (1, lm.n_q, T0), generator=torch.Generator().manual_seed(seed))


def _long(lm, rid, plan, prompt=None):
    """A request of several windows, as ContinuousGenerator.submit builds it (its seed is its window index)."""
    def make(k, p):
        cols = prefill_columns(lm, p.shape[-1], plan[k].length) if p is not None else 0
        return Request(plan[k].length, None, p, seed=k, id=rid, prefill_cols=cols, chain=chain)
    chain = WindowChain(plan, make, prompt)
    return chain.make(0, prompt)


def _poll_all(sched):
    out, polls = {}, 0
    while sched.pending:
        for req, codes in sched.poll():
            out[req.id] = codes
        polls += 1
    return out, polls


def test_slot_starts_at_its_prefilled_column(monkeypatch):
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    lm = FakeLM()
    sess = PrefillSession(lm, 2)
    sched = ContinuousScheduler(sess, 2)
    p = _prompt(lm, 9, 1)
    r = Request(20, None, p, id=0, prefill_cols=prefill_columns(lm, 9, 20))
    assert r.prefill_cols == 9
    sched.submit(r)
    sched.submit(Request(20, None, p, id=1))   # teacher-forced: starts at 0
    sched.poll()
    S = 20 + 3 + 1
    assert sched.steps_run == S - 1 - 9 and sess.state[0][1] != SLOT_ACTIVE and sched.pos == {1: S - 1 - 9}
    out, _ = _poll_all(sched)
    assert torch.equal(out[1][..., :9], p)
    monkeypatch.setenv('ACB_LM_PREFILL', '0')
    assert prefill_columns(lm, 9, 20) == 0
    monkeypatch.delenv('ACB_LM_PREFILL')
    assert prefill_columns(lm, 1, 20) == 0 and prefill_columns(lm, 2, 20) == 2   # the pass threshold: first >= 2


def test_next_window_is_readmitted_into_its_slot_ahead_of_the_queue():
    lm = FakeLM()
    sess = PrefillSession(lm, 2)
    sched = ContinuousScheduler(sess, 2)
    plan = window_plan(2.5, 1.0, 0.4, 20)   # windows of 20 frames striding by 8
    assert len(plan) == 5
    sched.submit(_long(lm, 0, plan))
    for i in range(1, 6):
        sched.submit(Request(7 + i, None, None, id=i))
    out, _ = _poll_all(sched)
    admits = [e for e in sess.log if e[0] == 'admit']
    assert [a[2] for a in admits if a[2] != 0] == [1, 2, 3, 4, 5], 'a waiting request overtook another'
    assert [a[1] for a in admits if a[2] == 0] == [0] * 5, 'a later window left its slot'
    # each re-admission follows its window's finish in the same poll: no step and no other admission in between
    for j, e in enumerate(sess.log):
        if e[0] == 'admit' and e[2] == 0 and j > 0:
            assert sess.log[j - 1][0] == 'steps'
    assert sched.readmitted == 4
    assert out[0].shape == (1, 4, 50)
    assert torch.equal(out[0][..., :20], sess.codes(lm, Request(20, id=0)))


def test_tight_pool_hands_pages_to_the_next_window():
    lm = FakeLM()
    need = PagePool.need(20 + 3 + 1)
    sess = PagedPrefillSession(lm, 3, 2 * need)   # two requests of the longest length at a time
    sched = ContinuousScheduler(sess, 3)
    plan = window_plan(2.5, 1.0, 0.4, 20, 5)
    sched.submit(Request(20, None, None, id=0))
    sched.submit(_long(lm, 1, plan, _prompt(lm, 5, 2)))
    for i in range(2, 7):
        sched.submit(Request(20, None, None, id=i))
    out, _ = _poll_all(sched)
    assert sorted(out) == list(range(7)) and out[1].shape == (1, 4, 50)
    pages = [e for e in sess.log if e[0] == 'pages' and e[2] == 1]
    assert len(pages) == len(plan)
    for a, b in zip(pages, pages[1:]):
        assert b[1] == a[1] and set(b[3]) <= set(a[3]), 'a later window took pages it did not release'
    firsts = [e[2] for e in sess.log if e[0] == 'admit']
    firsts = [rid for k, rid in enumerate(firsts) if rid not in firsts[:k]]
    assert firsts == list(range(7)), 'a waiting request overtook another'
    assert sched.page_wait_steps > 0 and sess.pages.in_use == 0


@pytest.mark.parametrize('when', ['waiting', 'first window', 'between windows', 'last window'])
def test_cancel_a_long_request(when):
    lm = FakeLM()
    sess = PagedPrefillSession(lm, 1, PagePool.need(24) * 2)
    sched = ContinuousScheduler(sess, 1, poll_steps=5)
    plan = window_plan(2.5, 1.0, 0.4, 20)
    sched.submit(Request(10, None, None, id=9))
    sched.submit(_long(lm, 0, plan))
    sched.submit(Request(10, None, None, id=1))

    def due():
        if when == 'waiting':
            return any(r.id == 0 for r in sched.waiting)
        r = sched.active.get(0)
        if r is None or r.id != 0:
            return False
        k = r.chain.k
        return {'first window': k == 0, 'between windows': k == 1 and sched.pos[0] == r.prefill_cols,
                'last window': k == len(plan) - 1}[when]

    got, cancelled = {}, False
    while sched.pending:
        if not cancelled and due():
            assert sched.cancel(0) and not sched.cancel(0)
            assert 0 not in [r.id for r in sched.active.values()] and 0 not in [r.id for r in sched.waiting]
            cancelled = True
        for req, codes in sched.poll():
            got[req.id] = codes
    assert cancelled and sorted(got) == [1, 9] and sess.pages.in_use == 0
    if when == 'between windows':   # the poll before the cancel finished window 0 and admitted window 1
        assert [e[2] for e in sess.log if e[0] == 'admit'].count(0) == 2


class IdentityDecoder:
    """A stream decoder whose audio is codebook 0 of the frames it is pushed, as float."""

    def __init__(self, n):
        self.n = n

    def push(self, codes):
        assert codes.shape[0] == self.n
        return codes[:, :1].float()

    def flush(self):
        return torch.zeros(self.n, 1, 0)

    def select(self, items):
        return IdentityDecoder(len(items))


def test_cohorts_with_mixed_start_columns():
    lm = FakeLM()
    sess = PrefillSession(lm, 4)
    sched = ContinuousScheduler(sess, 4, poll_steps=3)
    stream = CohortStream(sched, IdentityDecoder, sess.max_delay)
    reqs = [Request(30, None, _prompt(lm, 12, 1), id=0, prefill_cols=12), Request(25, None, None, id=1),
            Request(30, None, _prompt(lm, 12, 2), id=2, prefill_cols=12), Request(40, None, _prompt(lm, 33, 3), id=3,
                                                                                  prefill_cols=33),
            Request(20, None, _prompt(lm, 5, 4), id=4, prefill_cols=5)]
    for r in reqs:
        sched.submit(r)
    pieces = {r.id: [] for r in reqs}
    finals = set()
    first = stream.poll()
    assert sorted(co.col0 for co in stream.cohorts) == [0, 12, 33], 'one cohort per start column'
    for ev in first:
        pieces[ev[0]].append(ev)
    early = {rid: sum(e[2].shape[-1] for e in evs) for rid, evs in pieces.items()}
    assert early[3] == 33 + 3 - sess.max_delay and early[0] == 12 + 3 - sess.max_delay and early[1] == 0
    while sched.pending:
        for ev in stream.poll():
            assert ev[0] not in finals
            pieces[ev[0]].append(ev)
            if ev[3]:
                finals.add(ev[0])
    assert finals == {0, 1, 2, 3, 4}
    for r in reqs:
        tok = torch.cat([e[2] for e in pieces[r.id]], dim=-1)
        wav = torch.cat([e[1] for e in pieces[r.id]], dim=-1)
        want = sess.codes(lm, r)
        assert torch.equal(tok, want) and torch.equal(wav, want[:, :1].float()), f'request {r.id}'


# ----------------------------------------------------------------------------- submit: seeds, refusals

def _gen_model(melody):
    """A model whose conditions draw from torch's generator, so the order of condition and seed draws shows."""
    calls = []

    def conditions(attrs):
        calls.append(attrs)
        torch.rand(1)
        return None, (torch.zeros(2, 5, 8) if melody else None)

    lm = FakeLM()
    lm.cross_attention, lm.has_prefix, lm.cfg_coef, lm._condition_tensors = not melody, melody, 3.0, conditions
    m = types.SimpleNamespace(lm=lm, duration=1.0, max_duration=1.0, extend_stride=0.4, frame_rate=20,
                              _has_melody=melody, _prepare_tokens_and_attributes=lambda d, p: (['a'], None),
                              _window_attributes=lambda attrs, offset: [('w', offset)])
    return m, calls


def _bare_generator(m, prefill=True, stream=None):
    gen = ContinuousGenerator.__new__(ContinuousGenerator)
    gen.model, gen.prefill_prompts, gen.stream = m, prefill, stream
    gen.defaults = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0)
    gen.session = types.SimpleNamespace(max_text=8, max_prefix=8)
    gen.scheduler = types.SimpleNamespace(submitted=[])
    gen.scheduler.submit = gen.scheduler.submitted.append
    gen._ids = itertools.count()
    return gen


@pytest.mark.parametrize('melody', [False, True])
def test_submit_draws_one_seed_per_window_in_generate_order(melody):
    m, calls = _gen_model(melody)
    gen = _bare_generator(m)
    torch.manual_seed(7)
    gen.submit('x', duration=2.5)
    plan = window_plan(2.5, 1.0, 0.4, 20)
    # generate: each window computes its conditions (here one draw) and then draws its seed
    torch.manual_seed(7)
    want = []
    for _ in plan:
        torch.rand(1)
        want.append(int(torch.randint(0, 2 ** 62, (1,)).item()))
    if not melody:   # a text condition is computed once: the draws are the seeds, one per window
        torch.manual_seed(7)
        torch.rand(1)
        want = [int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in plan]
    (req,) = gen.scheduler.submitted
    chain = req.chain
    seeds = [req.seed] + [chain.make(k, None).seed for k in range(1, len(plan))]
    assert seeds == want and len(set(seeds)) == len(plan)
    assert [w.length for w in plan] == [req.max_gen_len] + [chain.make(k, None).max_gen_len for k in range(1, len(plan))]
    if melody:   # each window's melody is re-sliced from its offset
        assert calls == [[('w', w.time_offset)] for w in plan]
    # a request within max_duration draws one seed, as before
    torch.manual_seed(7)
    gen.submit('x', duration=0.5)
    assert gen.scheduler.submitted[-1].chain is None


def test_extension_refusals_before_device_work():
    m, _ = _gen_model(False)
    m._prepare_tokens_and_attributes = _no_device
    with pytest.raises(NotImplementedError, match='max_duration'):
        _bare_generator(m, prefill=False).submit('x', duration=1.3)
    with pytest.raises(NotImplementedError, match='chunk_duration'):
        _bare_generator(m, stream=object()).submit('x', duration=1.3)
    with pytest.raises(AssertionError, match='device work'):   # within max_duration the same call reaches the conditions
        _bare_generator(m, stream=object()).submit('x', duration=1.0)


def test_header_declares_admit_prompt():
    import os
    from audiocraft_b200 import _lib
    from tests import helpers as H
    header = open(os.path.join(H.ROOT, 'include', 'audiocraft_b200.h')).read()
    assert 'acb_lm_admit_prompt' in _lib.EXPORTS and 'int acb_lm_admit_prompt(' in header
