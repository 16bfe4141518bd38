"""Paged continuous batching on the host: the page accounting of `batching.PagePool` under `ContinuousScheduler` against a fake
device session that takes and returns pages where `SlotSession` does (admission, `collect`, `retire`); FIFO order with the
head request waiting for pages; the refusal of a pool that cannot hold one request of the longest length; the
`kv_cache_gb` -> pages arithmetic; and every refusal before device work."""
import contextlib
import math
import types

import pytest
import torch

from audiocraft_b200 import _lib
from audiocraft_b200.batching import (ContinuousGenerator, ContinuousScheduler, PagePool, Request, SlotSession,
                                      kv_page_bytes, kv_pages_for_budget, pattern_sequence)
from tests.test_continuous_serving_host import FakeLM, FakeSession

PAGE = _lib.ACB_LM_KV_PAGE


class FakePagedSession(FakeSession):
    """FakeSession with a page pool: admission takes the request's pages, `collect` and `retire` return them, as in
    `SlotSession(kv_pages=...)`.  `owner` maps every page a live slot holds to that slot, and admission asserts that no page
    is handed to two live slots."""

    def __init__(self, lm, slots, n_pages):
        super().__init__(lm, slots)
        self.pages = PagePool(n_pages)
        self.owner = {}
        self.admitted = []

    def positions(self, req):
        return (0 if req.prefix is None else req.prefix.shape[1]) + pattern_sequence(self.lm, None, req.max_gen_len)[0].shape[-1]

    def admit(self, slot, req):
        super().admit(slot, req)
        for p in self.pages.take(slot, self.positions(req)):
            assert p not in self.owner, f'page {p} handed to slot {slot} while slot {self.owner.get(p)} holds it'
            self.owner[p] = slot
        self.admitted.append(req.id)

    def _free(self, slot):
        for p in self.pages.held.get(slot, []):
            del self.owner[p]
        self.pages.release(slot)

    def retire(self, slot):
        super().retire(slot)
        self._free(slot)

    def collect(self, slot, req):
        self._free(slot)
        return super().collect(slot, req)


def _req(n, P, rid):
    return Request(n, None, None, seed=rid, id=rid, prefix=None if P is None else torch.zeros(2, P, 1))


def _check_pool(sess, sched):
    pool = sess.pages
    assert 0 <= pool.in_use <= pool.n_pages
    held = [p for ids in pool.held.values() for p in ids]
    assert len(held) == len(set(held)) == pool.in_use, 'a page is held twice'
    assert sorted(held + pool.free) == list(range(pool.n_pages)), 'a page is lost or duplicated'
    assert set(pool.held) == set(sched.active), 'pages held by a slot that is not decoding, or a slot without pages'
    for slot, req in sched.active.items():
        assert len(pool.held[slot]) == PagePool.need(sess.positions(req))


def test_page_counts():
    assert [PagePool.need(n) for n in (1, 63, 64, 65, 128, 129)] == [2, 2, 2, 4, 4, 6]


def test_page_accounting_with_finishes_and_cancellations():
    lm = FakeLM()
    slots, n_pages = 6, 14
    sess = FakePagedSession(lm, slots, n_pages)
    sched = ContinuousScheduler(sess, slots, poll_steps=7)
    g = torch.Generator().manual_seed(0)
    reqs = []
    for i in range(60):
        n = int(torch.randint(1, 200, (1,), generator=g))
        P = [None, 0, 1, 63, 64, 100][i % 6]
        reqs.append(_req(n, P, i))
    for r in reqs:
        assert PagePool.need(sess.positions(r)) <= n_pages
        sched.submit(r)
    finished, cancelled = set(), set()
    polls = 0
    while sched.pending:
        for req, _ in sched.poll():
            finished.add(req.id)
        _check_pool(sess, sched)
        polls += 1
        if polls % 5 == 0 and sched.active:    # cancel a decoding request: its pages come back at once
            slot = min(sched.active)
            rid = sched.active[slot].id
            before = sess.pages.in_use
            assert sched.cancel(rid)
            cancelled.add(rid)
            assert sess.pages.in_use == before - PagePool.need(sess.positions(reqs[rid]))
            _check_pool(sess, sched)
        if polls % 7 == 0 and sched.waiting:   # a waiting request never held pages
            rid = sched.waiting[-1].id
            before = sess.pages.in_use
            assert sched.cancel(rid)
            cancelled.add(rid)
            assert sess.pages.in_use == before
    assert finished | cancelled == {r.id for r in reqs} and not finished & cancelled
    assert sess.pages.in_use == 0 and not sess.owner and len(sess.pages.free) == n_pages
    assert 0 < sess.pages.peak <= n_pages
    assert sched.page_steps <= sched.steps_run * n_pages


def test_fifo_head_waits_for_pages():
    """A long request at the head waits for pages with a slot free; a short request behind it, whose pages would fit, is not
    admitted before it, so the long request is not starved."""
    lm = FakeLM()
    S = lambda n: pattern_sequence(lm, None, n)[0].shape[-1]   # noqa: E731
    long_n = 100
    assert PagePool.need(S(long_n)) == 4 and PagePool.need(S(1)) == 2
    sess = FakePagedSession(lm, 4, 6)
    sched = ContinuousScheduler(sess, 4)
    sched.submit(_req(long_n, None, 0))   # 4 pages
    sched.submit(_req(long_n, None, 1))   # 4 pages: waits for request 0
    sched.submit(_req(1, None, 2))        # 2 pages would fit next to request 0, but it is behind request 1
    order = []
    while sched.pending:
        done = sched.poll()
        order += [r.id for _, r in sched.last_admitted]
        if 1 not in order:
            assert order == [0] and [r.id for r in sched.waiting] == [1, 2]
        _check_pool(sess, sched)
        assert all(r.id in (0, 1, 2) for r, _ in done)
    assert order == [0, 1, 2] == sess.admitted
    assert sched.page_wait_steps == S(long_n) - 1   # the head waited for request 0's whole decode


def test_contiguous_scheduler_keeps_its_order():
    """Without a page pool (a contiguous session) admission is FIFO into free slots, as before."""
    lm = FakeLM()
    sess = FakeSession(lm, 2)
    sched = ContinuousScheduler(sess, 2)
    for i in range(5):
        sched.submit(_req(3 + i, None, i))
    order = []
    while sched.pending:
        sched.poll()
        order += [r.id for _, r in sched.last_admitted]
    assert order == list(range(5)) and sched.page_wait_steps == 0 and sched.page_steps == 0


# ----------------------------------------------------------------------------- budget arithmetic and refusals

def test_kv_cache_gb_to_pages():
    medium = types.SimpleNamespace(num_layers=48, dim=1536)
    large = types.SimpleNamespace(num_layers=48, dim=2048)
    assert kv_page_bytes(medium) == 64 * 294912 and kv_page_bytes(large) == 64 * 393216
    assert kv_pages_for_budget(medium, 56.7) == math.floor(56.7e9 / (64 * 294912)) == 3004
    assert kv_pages_for_budget(large, 40) == math.floor(40e9 / (64 * 393216))
    assert kv_pages_for_budget(medium, 1) == 52   # 1e9 / 18874368 = 52.98
    for bad in (0, -1.0, float('nan'), float('inf'), True, '8', None):
        with pytest.raises(ValueError):
            kv_pages_for_budget(medium, bad)


class _RefusingLM(FakeLM):
    """An LM whose first device call fails the test."""

    def __init__(self):
        super().__init__()
        self.device, self.cfg_coef, self.cross_attention, self.num_layers, self.dim = None, 3.0, True, 2, 64

    def _ensure(self, *a, **k):
        raise AssertionError('device work before the refusal')


def test_pool_that_cannot_hold_one_request_is_refused_before_device_work(monkeypatch):
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    lm = _RefusingLM()
    S = pattern_sequence(lm, None, 100)[0].shape[-1]
    need = PagePool.need(S)
    for bad in (need - 1, 0, 1, True, 2.5):
        with pytest.raises(ValueError):
            SlotSession(lm, 4, 100, kv_pages=bad)
    with pytest.raises(AssertionError, match='device work'):   # the smallest pool that holds one request gets to the device
        SlotSession(lm, 4, 100, kv_pages=need)
    # with a condition prefix bound the longest request is max_prefix + S positions
    lm.has_prefix = True
    need_p = PagePool.need(70 + S)
    with pytest.raises(ValueError):
        SlotSession(lm, 4, 100, max_prefix=70, kv_pages=need_p - 1)
    with pytest.raises(AssertionError, match='device work'):
        SlotSession(lm, 4, 100, max_prefix=70, kv_pages=need_p)


def _fake_model():
    lm = _RefusingLM()
    gp = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0, two_step_cfg=False, cfg_coef_beta=None)
    return types.SimpleNamespace(lm=lm, generation_params=gp, max_duration=2.0, duration=1.0, frame_rate=50,
                                 _has_melody=False)


def test_generator_budget_refusals_before_device_work(monkeypatch):
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    m = _fake_model()
    for bad in (0, -3, float('nan'), True):
        with pytest.raises(ValueError, match='kv_cache_gb'):
            ContinuousGenerator(m, slots=4, kv_cache_gb=bad)
    page = kv_page_bytes(m.lm)
    need = PagePool.need(pattern_sequence(m.lm, None, 100)[0].shape[-1])   # max_duration 2 s at 50 Hz: 100 frames
    with pytest.raises(ValueError, match='cannot hold one request'):
        ContinuousGenerator(m, slots=4, kv_cache_gb=(need - 1) * page / 1e9)
    with pytest.raises(AssertionError, match='device work'):
        ContinuousGenerator(m, slots=4, kv_cache_gb=(need + 0.5) * page / 1e9)


def test_generator_passes_the_page_count(monkeypatch):
    seen = {}

    def fake_init(self, lm, slots, max_gen_len, max_text, **kw):
        seen.update(kw, slots=slots)
        raise AssertionError('device work')

    monkeypatch.setattr(SlotSession, '__init__', fake_init)
    m = _fake_model()
    with pytest.raises(AssertionError):
        ContinuousGenerator(m, slots=96, kv_cache_gb=1.0)
    assert seen['kv_pages'] == kv_pages_for_budget(m.lm, 1.0) and seen['slots'] == 96
    with pytest.raises(AssertionError):
        ContinuousGenerator(m, slots=8)
    assert seen['kv_pages'] is None


def test_header_declares_the_paged_calls():
    import os
    from tests import helpers as H
    header = open(os.path.join(H.ROOT, 'include', 'audiocraft_b200.h')).read()
    assert f'#define ACB_LM_KV_PAGE {PAGE}' in header
    assert f'#define ACB_LM_MAX_PAGES_PER_ROW {_lib.ACB_LM_MAX_PAGES_PER_ROW}' in header
    assert _lib.ACB_LM_MAX_PAGES_PER_ROW == math.ceil(12000 / PAGE)
    for name in ('acb_lm_begin_slots_paged', 'acb_lm_admit_paged'):
        assert name in _lib.EXPORTS and name in header
