"""GPU: continuous batching with prefilled prompts and window extension (`continuous(prefill_prompts=True)`,
acb_lm_admit_prompt).

* LM level, at 4 and 32 slots (mma.sync GEMMs), greedy and sampled: requests whose prompts prefill 0 (1 frame), 2, 3, 31,
  32, 33, 65 and max_gen_len - 1 columns, mixed with unprompted ones and reusing slots, are bit-identical to
  `LMModel.generate` of each alone with the default prefill.  A paged session with a tight pool gives the same tokens.  At
  40 slots (wide GEMM) paged equals contiguous bit for bit, and greedy results equal `generate` up to argmax near-ties.
* Admission K/V: after one admission of a request with a condition prefix and a prefilled prompt, the K/V of every prefix and
  prompt position gathered from the slot's pages equal the contiguous session's rows, which equal `generate` alone.
* Public path, max_duration 1 s and extend_stride 0.4 s: short, continuation and longer-than-max_duration requests (with and
  without a prompt, melody requests on the mono and stereo melody models, AudioGen) at 4 slots, contiguous and paged with a
  pool that holds only a few requests, equal `generate` / `generate_continuation` / `generate_with_chroma` alone after the
  same seed.
* Streaming with prefilled prompts: the pieces concatenate to the non-streamed waveforms.
"""
import pytest
import torch

from audiocraft_b200.batching import ContinuousScheduler, PagePool, Request, SlotSession, kv_page_bytes, prefill_columns
from tests import helpers as H
from tests import test_gpu_continuous_melody as M
from tests.test_gpu_continuous import NEAR_TIE, WAV_TOL, _cross, _model, _prompt, _sequence
from tests.test_gpu_continuous_serving import _audiogen

pytestmark = pytest.mark.gpu

N = 90   # the LM-level session's max_gen_len


def _lm_requests(cfg, sd, m):
    """Prompted requests at the prefill thresholds and pass boundaries, with unprompted ones between them."""
    reqs = []
    for i, (n, T0) in enumerate([(40, 1), (20, 0), (50, 2), (45, 3), (60, 31), (33, 0), (70, 32), (80, 33), (N, 65),
                                 (N, N - 1), (12, 0), (66, 40)]):
        torch.manual_seed(500 + i)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        prompt = _prompt(cfg, T0, 900 + i)
        reqs.append(Request(n, _cross(cfg, sd, 1 + (7 * i) % 20, 40 + i), prompt, seed=seed, id=i,
                            prefill_cols=prefill_columns(m, T0, n) if T0 else 0))
    assert [r.prefill_cols for r in reqs[:10]] == [0, 0, 2, 3, 31, 0, 32, 33, 65, N - 1]
    return reqs


def _fresh(r):
    return Request(r.max_gen_len, r.cross, r.prompt, r.seed, r.id, prefill_cols=r.prefill_cols)


def _serve(m, slots, reqs, sampling, kv_pages=None):
    sess = SlotSession(m, slots, N, use_sampling=sampling, kv_pages=kv_pages)
    sched = ContinuousScheduler(sess, slots)
    for r in reqs:
        sched.submit(_fresh(r))
    got = {}
    while sched.pending:
        for r, codes in sched.poll():
            got[r.id] = codes.cpu()
    return got, sess


def _alone(m, r, sampling):
    torch.manual_seed(500 + r.id)
    return m.generate(None if r.prompt is None else r.prompt.cuda(), [], num_samples=1, max_gen_len=r.max_gen_len,
                      use_sampling=sampling, temp=1.0, top_k=250, top_p=0.0, cross_attention_src=r.cross).cpu()


@pytest.mark.parametrize('sampling', [False, True])
@pytest.mark.parametrize('slots', [4, 32, 40])
def test_prefilled_session_equals_generate_alone(slots, sampling, monkeypatch):
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    monkeypatch.delenv('ACB_LM_PREFILL_PER', raising=False)
    cfg, sd, m = _model('lm_mini')
    reqs = _lm_requests(cfg, sd, m)
    got, _ = _serve(m, slots, reqs, sampling)
    longest = PagePool.need(N + 4)
    paged, sess = _serve(m, slots, reqs, sampling, kv_pages=3 * longest)
    assert sess.pages.peak <= 3 * longest
    for r in reqs:
        assert torch.equal(paged[r.id], got[r.id]), f'request {r.id}: paged tokens differ from the contiguous session'
    margins = []
    for r in reqs:
        if slots > 32 and sampling:
            continue   # the wide GEMM sums in another order: only the greedy run is held to generate (near-tie rule)
        want = _alone(m, r, sampling)
        if r.prompt is not None:
            assert torch.equal(got[r.id][..., :r.prompt.shape[-1]], r.prompt)
        if slots <= 32:
            assert torch.equal(got[r.id], want), f'request {r.id} (prefill {r.prefill_cols}) differs from generate alone'
        elif not torch.equal(got[r.id], want):
            seq = _sequence(m, got[r.id])
            lg = m.teacher_forced_logits(seq, r.cross, m.cfg_coef).cpu()
            step = int((seq != _sequence(m, want)).any(0).any(0).nonzero()[0])
            top2 = lg[step - 1].topk(2, dim=-1).values
            margin = (top2[..., 0] - top2[..., 1]).min().item()
            assert margin < NEAR_TIE, f'request {r.id}: differs at step {step} with argmax margin {margin:.3e}'
            margins.append(margin)
    print(f'slots={slots} sampling={sampling}: {len(reqs)} requests, paged == contiguous, near-ties {margins}')


@pytest.mark.parametrize('pe', ['sin', 'rope'])
def test_admission_kv_pages_equal_contiguous_rows(pe, monkeypatch):
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    monkeypatch.delenv('ACB_LM_PREFILL_PER', raising=False)
    cfg, sd, m = M._model(pe, True)
    slots, s, n, P, T0 = 4, 2, 120, 37, 70
    req = M._req(cfg, sd, n, P, 9, T0, 5, 9, 1)
    req.prefill_cols = prefill_columns(m, T0, n)
    assert req.prefill_cols == T0
    pos = P + req.prefill_cols

    def admitted(kv_pages=None):
        sess = SlotSession(m, slots, n, max_prefix=M.MAX_PREFIX, kv_pages=kv_pages)
        for k in (0, 1, 3):   # the other slots hold requests of their own
            sess.admit(k, M._req(cfg, sd, 40, [5, 60, 33][k % 3], 7, [0, 9, 3][k % 3], k, 10 + k, 50 + 10 * k))
        sess.steps(3)
        r = Request(req.max_gen_len, req.cross, req.prompt, req.seed, req.id, prefix=req.prefix,
                    prefill_cols=req.prefill_cols)
        sess.admit(s, r)
        torch.cuda.synchronize()
        assert sess.status()[s] == (req.prefill_cols, 1), 'the slot does not start at its prefilled column'
        return sess

    sess = admitted()
    b = m._bufs
    want_k = b['k_cache'][:, [s, slots + s], :, :pos].clone()
    want_v = b['v_cache'][:, [s, slots + s], :, :pos].clone()
    sess = admitted(kv_pages=PagePool.need(M.MAX_PREFIX + 200) * 4)
    ids = sess.pages.held[s]
    half = len(ids) // 2
    for j, rows in enumerate((ids[:half], ids[half:])):
        k = sess.k_pool[:, rows].permute(0, 2, 1, 3, 4).reshape(cfg['num_layers'], -1, len(rows) * 64, 64)[:, :, :pos]
        v = sess.v_pool[:, rows].permute(0, 2, 1, 3, 4).reshape(cfg['num_layers'], -1, len(rows) * 64, 64)[:, :, :pos]
        assert torch.equal(k, want_k[:, j]), f'row {j}: K in the pages differ from the contiguous session'
        assert torch.equal(v, want_v[:, j]), f'row {j}: V in the pages differ from the contiguous session'
    m.generate(req.prompt.cuda(), [], num_samples=1, max_gen_len=n, use_sampling=False, cross_attention_src=req.cross,
               prefix=req.prefix)
    b = m._bufs
    assert torch.equal(want_k, b['k_cache'][:, :2, :, :pos]), 'K of the admission differ from generate alone'
    assert torch.equal(want_v, b['v_cache'][:, :2, :, :pos]), 'V of the admission differ from generate alone'


# ----------------------------------------------------------------------------- public path: prompts and extension

SAMPLING = dict(use_sampling=True, top_k=50, temperature=1.0)


def _small(mg):
    mg.max_duration = 1.0
    mg.set_generation_params(extend_stride=0.4, **SAMPLING)
    return mg


def _budget(mg, requests):
    """A KV budget of about `requests` requests of the longest length."""
    from audiocraft_b200.batching import prefix_bound
    S = int(mg.max_duration * mg.frame_rate) + max(mg.lm.pattern_provider.delays) + 1
    return requests * PagePool.need(prefix_bound(mg.lm, 64) + S) * kv_page_bytes(mg.lm) / 1e9


def _run(mg, items, **kw):
    """items: [(i, (description, duration, melody, prompt))], request i submitted after torch.manual_seed(1000 + i)."""
    gen = mg.continuous(slots=4, return_tokens=True, prefill_prompts=True, **kw)
    ids = {}
    for i, (desc, dur, melody, prompt) in items:
        torch.manual_seed(1000 + i)
        ids[gen.submit(desc, duration=dur, melody=melody, melody_sample_rate=None if melody is None else 32000,
                       prompt=prompt, prompt_sample_rate=None if prompt is None else mg.sample_rate)] = i
    got = {}
    if kw.get('chunk_duration') is None:
        for rid, wav, tok in gen.run():
            got[ids[rid]] = (wav, tok)
    else:
        pieces = {}
        for rid, piece, tok, final in gen.run():
            pieces.setdefault(ids[rid], []).append((piece, tok))
        for i, ps in pieces.items():
            got[i] = (torch.cat([p for p, _ in ps], -1), torch.cat([t for _, t in ps], -1))
    assert sorted(got) == sorted(i for i, _ in items)
    return got, gen


def _check_public(mg, reqs, monkeypatch):
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    got, gen = _run(mg, list(enumerate(reqs)))
    assert gen.scheduler.readmitted > 0
    paged, pgen = _run(mg, list(enumerate(reqs)), kv_cache_gb=_budget(mg, 2.5))
    worst = 0.0
    for i, (desc, dur, melody, prompt) in enumerate(reqs):
        mg.set_generation_params(duration=dur, extend_stride=0.4, **SAMPLING)
        torch.manual_seed(1000 + i)
        if melody is not None:
            wav, tok = mg.generate_with_chroma([desc], melody, 32000, return_tokens=True)
        elif prompt is not None:
            wav, tok = mg.generate_continuation(prompt, mg.sample_rate, [desc], return_tokens=True)
        else:
            wav, tok = mg.generate([desc], return_tokens=True)
        gw, gt = got[i]
        assert gt.shape == (1, mg.lm.n_q, int(dur * mg.frame_rate))
        assert torch.equal(gt, tok), f'request {i} ({dur} s): tokens differ from generate alone'
        assert torch.equal(paged[i][1], gt), f'request {i}: paged tokens differ from the contiguous session'
        assert gw.shape == wav.shape, (i, gw.shape, wav.shape)
        worst = max(worst, (gw - wav).abs().max().item(), (paged[i][0] - wav).abs().max().item())
    mg.set_generation_params(extend_stride=0.4, **SAMPLING)
    print(f'{mg.name}: {len(reqs)} requests, {gen.scheduler.readmitted} window re-admissions, occupancy '
          f'{gen.occupancy:.2f}; paged: {pgen.session.pages.n_pages} pages, {pgen.scheduler.page_wait_steps} steps with the '
          f'head waiting for pages; max |wav - alone| {worst:.2e}')
    assert worst <= WAV_TOL
    return got


def _text_requests(mg, channels=1):
    prompt = H.audio_input(dict(sample_rate=mg.sample_rate, channels=channels), 1, mg.sample_rate // 5, 3)[0]
    long_prompt = H.audio_input(dict(sample_rate=mg.sample_rate, channels=channels), 1, int(mg.sample_rate * 0.7), 4)[0]
    return [('a tune', 0.5, None, None), ('piano', 0.8, None, prompt), ('long one', 1.3, None, None),
            (None, 2.5, None, long_prompt), ('drums', 0.3, None, None), ('strings', 2.5, None, None),
            (None, 0.9, None, long_prompt), ('bass', 1.7, None, prompt)]


def test_musicgen_prompts_and_extension(monkeypatch):
    from audiocraft_b200.musicgen import MusicGen
    mg = _small(MusicGen.get_pretrained('synthetic/small'))
    reqs = _text_requests(mg)
    got = _check_public(mg, reqs, monkeypatch)
    # streamed with prefilled prompts (no extension): pieces of requests admitted together at different start columns
    short = [(i, r) for i, r in enumerate(reqs) if r[1] <= mg.max_duration]
    streamed, _ = _run(mg, short, chunk_duration=0.2)
    for i, _ in short:
        assert torch.equal(streamed[i][1], got[i][1]), f'request {i}: streamed tokens differ'
        torch.testing.assert_close(streamed[i][0], got[i][0], rtol=0, atol=1e-5)


def test_stereo_musicgen_prompts_and_extension(monkeypatch):
    from audiocraft_b200.musicgen import MusicGen
    mg = _small(MusicGen.get_pretrained('synthetic/stereo-small'))
    _check_public(mg, _text_requests(mg, channels=2)[:6], monkeypatch)


def test_audiogen_prompts_and_extension(monkeypatch):
    ag = _audiogen()
    ag.max_duration = 1.0
    ag.set_generation_params(extend_stride=0.4, **SAMPLING)
    _check_public(ag, _text_requests(ag), monkeypatch)


def _melody_requests(channels):
    mel = M._melody
    return [('d0', 1.3, mel(0.8, 1, channels), None), ('d1', 0.5, None, None), (None, 2.5, mel(2.0, 2, channels), None),
            ('d1', 0.6, mel(0.5, 3, channels), None), (None, 1.8, None, None), ('d0', 2.2, mel(3.1, 4, channels), None)]


def test_melody_extension(monkeypatch):
    _, _, _, mg = M._golden_musicgen()
    _check_public(_small(mg), _melody_requests(1), monkeypatch)


def test_stereo_melody_extension(monkeypatch):
    mg = _small(M._stereo_melody_musicgen())
    _check_public(mg, _melody_requests(2), monkeypatch)
