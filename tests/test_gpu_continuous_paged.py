"""GPU: paged continuous batching (`SlotSession(kv_pages=...)`, `continuous(kv_cache_gb=...)`, acb_lm_begin_slots_paged).

* A paged session and a contiguous one serve the same mixed requests (durations, continuation prompts, per-request sampling,
  a cancellation) at 4 slots (mma.sync GEMMs) and 40 slots (wide GEMM), sin and rope, with a pool smaller than slots x the
  longest request, so admissions wait and pages are reused: tokens and per-step CFG-mixed logits are bit-identical per
  request.  Between polls every page the host lists as free is overwritten with NaN, so a slot reading a page it does not
  own, or a position it has not written, would show.
* Page boundaries: requests of 63, 64, 65 and 128 positions, and condition prefixes of 63, 64 and 65 positions.
* Melody admission: the prefix K/V gathered from the slot's pages equal the contiguous session's rows bit for bit; the public
  `submit(melody=...)` path returns the same tokens and waveforms with a budget as without; streamed pieces concatenate to
  the paged session's waveforms.
* Handle handover: `generate` after a paged session equals a fresh model; the contiguous entry points refuse a paged handle
  and bad page lists are refused before any launch.
* Full size: synthetic MusicGen-medium, max_duration 10 s, 128 slots, half the contiguous reservation: tokens equal the
  contiguous session's.
"""
import ctypes as C
import math

import pytest
import torch

from audiocraft_b200 import _lib
from audiocraft_b200.batching import ContinuousScheduler, PagePool, Request, SlotSession, kv_page_bytes, pattern_sequence
from tests.test_gpu_continuous import _cross, _model, _prompt
from tests import test_gpu_continuous_melody as M

pytestmark = pytest.mark.gpu

PAGE = _lib.ACB_LM_KV_PAGE
WAV_TOL = 1e-4


class Recorder:
    """A device session for ContinuousScheduler that runs each step through step_logits and keeps every request's per-step
    CFG-mixed logits; with `nan_free`, every page the pool lists as free is overwritten with NaN before each poll's
    admissions (`before_poll`)."""

    def __init__(self, sess, nan_free=False):
        self.s, self.nan_free = sess, nan_free
        self.pages = sess.pages
        self.logits, self.live = {}, {}

    def positions(self, req):
        return self.s.positions(req)

    def before_poll(self):
        if self.nan_free and self.pages is not None and self.pages.free:
            idx = torch.tensor(self.pages.free, device=self.s.k_pool.device)
            self.s.k_pool[:, idx] = float('nan')
            self.s.v_pool[:, idx] = float('nan')

    def admit(self, slot, req):
        self.s.admit(slot, req)
        self.live[slot] = req
        self.logits[req.id] = []

    def retire(self, slot):
        self.s.retire(slot)
        del self.live[slot]

    def collect(self, slot, req):
        del self.live[slot]
        return self.s.collect(slot, req)

    def status(self):
        return self.s.status()

    def steps(self, n):
        for _ in range(n):
            lg = self.s.step_logits()
            for slot, req in self.live.items():
                self.logits[req.id].append(lg[slot].clone())


def _serve(sess, reqs, cancel=None, nan_free=False, poll_steps=None):
    """Serve reqs through ContinuousScheduler; `cancel` = (request id, polls after its admission).  Returns ({id: codes},
    {id: logits [steps, K, card]}, scheduler)."""
    rec = Recorder(sess, nan_free)
    sched = ContinuousScheduler(rec, sess.slots, poll_steps)
    for r in reqs:
        sched.submit(r)
    codes, admitted_at, polls = {}, {}, 0
    while sched.pending:
        rec.before_poll()
        for r, c in sched.poll():
            codes[r.id] = c.cpu()
        polls += 1
        for _, r in sched.last_admitted:
            admitted_at[r.id] = polls
        if cancel is not None and admitted_at.get(cancel[0]) == polls - cancel[1] + 1 and cancel[0] not in codes:
            assert sched.cancel(cancel[0])
            cancel = None
        if sess.pages is not None:
            held = [p for ids in sess.pages.held.values() for p in ids]
            assert len(held) == len(set(held)) == sess.pages.in_use
    if sess.pages is not None:
        assert sess.pages.in_use == 0, 'pages not returned'
    return codes, {k: torch.stack(v) for k, v in rec.logits.items() if v}, sched


def _compare(got, want, skip=()):
    (gc, gl), (wc, wl) = got, want
    assert set(gc) == set(wc)
    for rid in wc:
        assert torch.equal(gc[rid], wc[rid]), f'request {rid}: tokens differ'
    for rid in wl:
        if rid in skip:
            continue
        assert gl[rid].shape == wl[rid].shape, (rid, gl[rid].shape, wl[rid].shape)
        assert torch.equal(gl[rid], wl[rid]), f'request {rid}: logits differ by {(gl[rid] - wl[rid]).abs().max():.3e}'


def _mixed(cfg, sd, max_len, n_req, seed):
    g = torch.Generator().manual_seed(seed)
    opts = [dict(), dict(use_sampling=False), dict(top_k=5, temp=0.7), dict(top_p=0.9, top_k=0), dict(cfg_coef=1.0, temp=1.3)]
    reqs = []
    for i in range(n_req):
        n = [max_len, 2, 30, 61, 45, max_len - 7][i % 6]
        T0 = [0, 0, 5, 0, 11, 0][i % 6] if n > 12 else 0
        reqs.append(Request(n, _cross(cfg, sd, [1, 9, 30, 60][i % 4], 100 + i), _prompt(cfg, T0, 200 + i),
                            seed=int(torch.randint(0, 2 ** 62, (1,), generator=g)), id=i, **opts[i % 5]))
    return reqs


@pytest.mark.parametrize('pe', ['sin', 'rope'])
@pytest.mark.parametrize('slots', [4, 40])
def test_paged_session_equals_contiguous(slots, pe):
    cfg, sd, m = _model('lm_mini', pe)
    max_len = 120   # S = 124 positions: 2 pages per row
    n_req = 12 if slots == 4 else 70
    cancel = (3, 2)   # request 3 (61 frames) is cancelled 2 polls of at most 8 steps after its admission
    want = _serve(SlotSession(m, slots, max_len, top_k=20), _mixed(cfg, sd, max_len, n_req, 1), cancel, poll_steps=8)
    longest = PagePool.need(pattern_sequence(m, None, max_len)[0].shape[-1])
    n_pages = longest * (slots // 2) + 2   # half the slots' worth of the longest request: admissions wait for pages
    sess = SlotSession(m, slots, max_len, top_k=20, kv_pages=n_pages)
    got_c, got_l, sched = _serve(sess, _mixed(cfg, sd, max_len, n_req, 1), cancel, nan_free=True, poll_steps=8)
    _compare((got_c, got_l), want[:2], skip={cancel[0]})
    assert cancel[0] not in got_c
    assert sched.page_wait_steps > 0, 'the pool never made an admission wait'
    assert sess.pages.peak <= n_pages
    print(f'slots={slots} {pe}: {n_req} requests bit-identical paged vs contiguous; pool {n_pages} pages, peak '
          f'{sess.pages.peak}, head waited {sched.page_wait_steps} steps, occupancy {sched.occupancy:.2f} vs '
          f'{want[2].occupancy:.2f}')


def test_page_boundaries():
    """Requests whose P + S is 63, 64, 65 and 128 positions, and condition prefixes of 63, 64 and 65 positions."""
    cfg, sd, m = _model('lm_mini', 'sin')
    S1 = pattern_sequence(m, None, 1)[0].shape[-1]   # S(n) = n + S1 - 1
    reqs = lambda: [Request(S - S1 + 1, _cross(cfg, sd, 7, S), None, seed=S, id=i)   # noqa: E731
                    for i, S in enumerate((63, 64, 65, 128))]
    assert [pattern_sequence(m, None, r.max_gen_len)[0].shape[-1] for r in reqs()] == [63, 64, 65, 128]
    want = _serve(SlotSession(m, 4, 128), reqs())
    sess = SlotSession(m, 4, 128, kv_pages=PagePool.need(128 + S1) + 2)
    _compare(_serve(sess, reqs(), nan_free=True)[:2], want[:2])
    # condition prefixes across the page boundary, on a prepend model; the last request has P + S = 64
    cfg, sd, pm = M._model('sin', True)
    preqs = lambda: [M._req(cfg, sd, n, P, 5, 0, 10 + P, i, 40 + P)   # noqa: E731
                     for i, (P, n) in enumerate(((63, 20), (64, 20), (65, 20), (1, 63 - S1 + 1)))]
    want = _serve(SlotSession(pm, 4, 70, max_prefix=70), preqs())
    sess = SlotSession(pm, 4, 70, max_prefix=70, kv_pages=PagePool.need(70 + 70 + S1) + 4)
    _compare(_serve(sess, preqs(), nan_free=True)[:2], want[:2])


def _gather(pool, table, row, P):
    """[L, H, P, 64] of cache positions [0, P) of `row`, read through its page table."""
    pos = torch.arange(P, device=table.device)
    return pool[:, table[row, pos // PAGE].long(), :, pos % PAGE].permute(1, 2, 0, 3)   # indexed dim first: [P, L, H, 64]


def test_melody_admission_kv_and_public_path():
    g, cfg, sd, mg = M._golden_musicgen()
    lm = mg.lm
    slots, s, P = 4, 2, 37
    cond = torch.randn(1, 9, lm.dim, generator=torch.Generator().manual_seed(2)) * 0.1
    cross = torch.cat([cond, torch.zeros_like(cond)]) if lm.cross_attention else None
    req = lambda: Request(30, cross, None, seed=5, id=9, prefix=M._prefix(cfg, P, 3))   # noqa: E731
    cont = SlotSession(lm, slots, 40, max_prefix=64)
    cont.admit(s, req())
    torch.cuda.synchronize()
    want_k = lm._bufs['k_cache'][:, [s, slots + s], :, :P].clone()
    want_v = lm._bufs['v_cache'][:, [s, slots + s], :, :P].clone()
    paged = SlotSession(lm, slots, 40, max_prefix=64, kv_pages=8 * PagePool.need(64 + pattern_sequence(lm, None, 40)[0].shape[-1]))
    assert lm._bufs['k_cache'] is None
    paged.admit(0, req())           # another slot first, so the target's pages are not the first ones
    paged.admit(s, req())
    torch.cuda.synchronize()
    for j, row in enumerate((s, slots + s)):
        assert torch.equal(_gather(paged.k_pool, paged.page_table, row, P), want_k[:, j]), 'K of the admitted prefix differ'
        assert torch.equal(_gather(paged.v_pool, paged.page_table, row, P), want_v[:, j]), 'V of the admitted prefix differ'
    # the public path, with and without a budget, and streamed
    mg.set_generation_params(**M.SAMPLING)
    reqs = M._public_requests(1, ('d0', 'd1'))
    page = kv_page_bytes(lm)

    def run(kv_cache_gb, chunk_duration=None):
        gen = mg.continuous(slots=4, return_tokens=True, chunk_duration=chunk_duration, kv_cache_gb=kv_cache_gb)
        ids = {}
        for i, (desc, dur, melody, prompt) in enumerate(reqs):
            torch.manual_seed(1000 + i)
            ids[gen.submit(desc, duration=dur, melody=melody, melody_sample_rate=None if melody is None else 32000,
                           prompt=prompt, prompt_sample_rate=None if prompt is None else mg.sample_rate)] = i
        got, pieces = {}, {}
        for ev in gen.run():
            if chunk_duration is None:
                got[ids[ev[0]]] = (ev[1], ev[2])
            else:
                pieces.setdefault(ids[ev[0]], []).append((ev[1], ev[2]))
        for i, ps in pieces.items():
            got[i] = (torch.cat([p for p, _ in ps], -1), torch.cat([t for _, t in ps], -1))
        return got, gen

    want, _ = run(None)
    probe = SlotSession(lm, 4, int(mg.max_duration * mg.frame_rate))   # the session continuous() makes: its longest request
    longest = probe.max_prefix + probe.seq_len_max
    budget = (2 * PagePool.need(longest) + 1.5) * page / 1e9   # two of the longest requests: admissions wait for pages
    got, gen = run(budget)
    assert gen.session.pages is not None and gen.session.pages.n_pages == 2 * PagePool.need(longest) + 1
    worst = 0.0
    for i in want:
        assert torch.equal(got[i][1], want[i][1]), f'request {i}: tokens differ with a KV budget'
        worst = max(worst, (got[i][0] - want[i][0]).abs().max().item())
    assert worst <= WAV_TOL, worst
    streamed, _ = run(budget, chunk_duration=0.2)
    for i in got:
        assert torch.equal(streamed[i][1], got[i][1]), f'request {i}: streamed tokens differ'
        torch.testing.assert_close(streamed[i][0], got[i][0], rtol=0, atol=1e-5)
    print(f'melody public path: {len(reqs)} requests equal with a budget of {budget * 1e3:.3f} MB, max |wav diff| {worst:.2e}')


def test_handover_and_refusals():
    cfg, sd, m = _model('lm_mini', 'sin')
    cross = _cross(cfg, sd, 9, 1)

    def greedy(model):
        return model.generate(None, [], num_samples=1, max_gen_len=30, use_sampling=False, cross_attention_src=cross).cpu()

    fresh = greedy(_model('lm_mini', 'sin')[2])
    reqs = lambda: [Request(30, cross, None, seed=3, id=0), Request(20, _cross(cfg, sd, 4, 2), None, seed=4, id=1)]  # noqa: E731
    base = _serve(SlotSession(m, 4, 40, kv_pages=12), reqs())
    # a paged session with refused calls in between continues bit-identically
    sess = SlotSession(m, 4, 40, kv_pages=12)
    lm, L = m, m._lib
    assert lm._bufs['k_cache'] is None
    INVALID = -1
    samp = _lib.LMSampling(0, 1.0, 0, 0.0, 3.0, 0, 0, 0.0)
    st = _lib.stream()
    c16 = cross.cuda().contiguous()
    # the contiguous entry points on a paged handle
    assert L.acb_lm_begin(lm._handle, c16.data_ptr(), 1, 2, 9, 30, C.byref(samp), st) == INVALID
    assert L.acb_lm_begin_prefix(lm._handle, c16.data_ptr(), None, 0, 1, 2, 9, 30, C.byref(samp), st) == INVALID
    assert L.acb_lm_prefill(lm._handle, 0, 2, st) == INVALID
    assert L.acb_lm_begin_slots(lm._handle, 4, 64, 40, C.byref(samp), st) == INVALID
    S = pattern_sequence(m, None, 30)[0].shape[-1]
    assert PagePool.need(S) == 2

    def ids(*v):
        return (C.c_int32 * len(v))(*v)

    for pages, what in ((ids(0), 'too few pages'), (ids(0, 12), 'page id out of range'), (ids(0, -1), 'negative page id'),
                        (ids(3, 3), 'page given twice'), (ids(0, 1, 2, 3), 'too many pages')):
        assert L.acb_lm_admit_paged(lm._handle, 1, c16.data_ptr(), 9, None, 0, S, C.c_uint64(1), None, pages, len(pages),
                                    st) == INVALID, what
    pre = torch.zeros(2, 8, cfg['dim'], device='cuda')
    assert L.acb_lm_admit_paged(lm._handle, 1, c16.data_ptr(), 9, pre.data_ptr(), 8, S, C.c_uint64(1), None, ids(0, 1), 2,
                                st) == INVALID, 'prefix longer than max_prefix (0)'
    assert L.acb_lm_admit(lm._handle, 1, c16.data_ptr(), 9, S, C.c_uint64(1), None, st) == INVALID
    assert L.acb_lm_admit_prefix(lm._handle, 1, c16.data_ptr(), 9, None, 0, S, C.c_uint64(1), None, st) == INVALID
    _compare(_serve(sess, reqs())[:2], base[:2])
    # a contiguous session's handle refuses the paged calls
    SlotSession(m, 4, 40)
    assert L.acb_lm_begin_slots_paged(lm._handle, 4, 64, 40, 0, c16.data_ptr(), c16.data_ptr(), 4, c16.data_ptr(), 1, None,
                                      None, C.byref(samp), st) == INVALID
    assert L.acb_lm_admit_paged(lm._handle, 0, c16.data_ptr(), 9, None, 0, S, C.c_uint64(1), None, ids(0, 1), 2, st) == INVALID
    # generate after a paged session rebuilds a contiguous handle
    SlotSession(m, 4, 40, kv_pages=12)
    assert torch.equal(greedy(m), fresh)


def test_full_size_medium_half_budget():
    from audiocraft_b200.loaders import load_lm_model
    lm = load_lm_model('synthetic/medium')
    slots, max_gen_len = 128, 500   # 10 s at 50 Hz
    n_req = 192

    def reqs():
        out = []
        for i in range(n_req):
            T = 4 + i % 29
            cond = torch.randn(1, T, lm.dim, generator=torch.Generator().manual_seed(i)) * 0.1
            out.append(Request([500, 100, 250, 400, 37][i % 5], torch.cat([cond, torch.zeros_like(cond)]), None,
                               seed=1000 + i, id=i))
        return out

    def serve(sess):
        sched = ContinuousScheduler(sess, slots)
        for r in reqs():
            sched.submit(r)
        got = {}
        while sched.pending:
            for r, c in sched.poll():
                got[r.id] = c.cpu()
        return got, sched

    want, _ = serve(SlotSession(lm, slots, max_gen_len))
    S = pattern_sequence(lm, None, max_gen_len)[0].shape[-1]
    n_pages = math.floor(2 * slots * S * 0.5 / PAGE)   # half the contiguous reservation of 2 * slots rows x S positions
    sess = SlotSession(lm, slots, max_gen_len, kv_pages=n_pages)
    got, sched = serve(sess)
    assert set(got) == set(want)
    for rid in want:
        assert torch.equal(got[rid], want[rid]), f'request {rid}: tokens differ'
    print(f'medium, 128 slots: {n_req} requests bit-identical with {n_pages} pages ({n_pages * kv_page_bytes(lm) / 1e9:.1f} GB, '
          f'peak {sess.pages.peak}); head waited {sched.page_wait_steps} steps')
