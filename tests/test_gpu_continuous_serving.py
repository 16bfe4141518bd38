"""GPU: continuous batching as a service -- per-request sampling options, cancellation, and audio streamed while requests decode.

* Sessions on lm_mini at 4 slots (8 rows, lm_gemm_kernel) and 40 slots (80 rows, the wide GEMM) with requests that mix greedy,
  top-k 5 / 250, top-p 0.9, temperatures 0.7 / 1.3 and cfg_coef 1 / 3 / 7: every request's tokens and per-step CFG-mixed logits
  are bit-identical to the same request alone in a session.  At 4 slots (the GEMM regime of one item) its logits also equal
  `teacher_forced_logits` with its own cfg_coef and its tokens `LMModel.generate` of it alone with those options
  (ACB_LM_PREFILL=0); the wide GEMM of 40 slots sums in another order.
* Cancellation: a request retired mid-decode leaves the other requests bit-identical to a run without it, and the freed slot
  takes a new request at the next step, which is bit-identical to itself alone.
* The public path, `continuous(slots=4, chunk_duration=0.2, return_tokens=True)` with per-request options on synthetic
  MusicGen-small (with a continuation), stereo MusicGen-small and an AudioGen model: tokens equal `generate` alone, the
  concatenated pieces equal the non-streamed session's waveform exactly and `generate`'s within the EnCodec tolerance, and a
  cancelled request yields nothing after the cancel.
* A GroupNorm codec refuses `continuous(chunk_duration=...)` before a session is made.
"""
import copy

import pytest
import torch

from audiocraft_b200 import synth
from audiocraft_b200.batching import Request, SlotSession
from tests import helpers as H
from tests.test_gpu_continuous import _cross, _model, _prompt, _sequence

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4

# (use_sampling, temp, top_k, top_p, cfg_coef)
OPTIONS = [(False, 1.0, 250, 0.0, 3.0), (True, 1.0, 5, 0.0, 3.0), (True, 1.0, 250, 0.0, 7.0), (True, 1.0, 0, 0.9, 3.0),
           (True, 0.7, 250, 0.0, 1.0), (True, 1.3, 250, 0.0, 3.0), (True, 0.7, 0, 0.9, 7.0), (False, 1.0, 0, 0.0, 1.0)]


def _opts(o):
    return dict(zip(('use_sampling', 'temp', 'top_k', 'top_p', 'cfg_coef'), o))


def _requests(cfg, sd):
    out = []
    for i, o in enumerate(OPTIONS):
        n = [30, 12, 25, 40, 9, 33, 18, 21][i]
        T = [9, 1, 30, 4, 60, 2, 17, 5][i]
        T0 = [0, 3, 0, 5, 0, 0, 2, 0][i]
        out.append(Request(n, _cross(cfg, sd, T, 300 + i), _prompt(cfg, T0, 400 + i), seed=1000 + 7 * i, id=i, **_opts(o)))
    return out


def _fresh(r):
    return Request(r.max_gen_len, r.cross, r.prompt, r.seed, r.id, use_sampling=r.use_sampling, temp=r.temp, top_k=r.top_k,
                   top_p=r.top_p, cfg_coef=r.cfg_coef)


def _drive(sess, events, n_total, cancels=None):
    """Run n_total steps through SlotSession.step_logits, admitting events[step] = [(slot, req)] and retiring the slots of
    cancels[step] before each step.  Returns ({id: codes}, {id: logits [n_steps, K, card]})."""
    logs, active, codes = {}, {}, {}
    for t in range(n_total):
        for slot in (cancels or {}).get(t, []):
            sess.retire(slot)
            del active[slot]
        for slot, req in events.get(t, []):
            assert slot not in active
            sess.admit(slot, req)
            active[slot] = req
            logs[req.id] = []
        if not active:
            continue
        lg = sess.step_logits()
        for slot, req in list(active.items()):
            logs[req.id].append(lg[slot].clone())
            if len(logs[req.id]) == req.meta['S'] - 1:
                codes[req.id] = sess.collect(slot, req)
                del active[slot]
    assert not active, 'n_total too small'
    assert all(st != 1 for _, st in sess.status())
    return codes, {k: torch.stack(v) for k, v in logs.items()}


@pytest.mark.parametrize('slots', [4, 40])
def test_mixed_options_equal_each_request_alone(slots, monkeypatch):
    cfg, sd, m = _model('lm_mini')
    reqs = _requests(cfg, sd)
    # a session whose own options none of the requests uses: every request samples with its own
    sess = SlotSession(m, slots, 48, use_sampling=True, temp=2.0, top_k=3, top_p=0.0, cfg_coef=0.5)
    if slots >= len(reqs):   # admitted at different steps into slots spread over the session
        ev = {}
        for i, r in enumerate(reqs):
            ev.setdefault([0, 0, 3, 3, 7, 11, 11, 20][i], []).append(((5 * i) % slots, _fresh(r)))
    else:                    # 4 slots: the last four reuse the first four's slots after they retire
        ev = {0: [(0, _fresh(reqs[0])), (1, _fresh(reqs[1])), (2, _fresh(reqs[2])), (3, _fresh(reqs[3]))],
              36: [(0, _fresh(reqs[4])), (1, _fresh(reqs[5]))], 46: [(2, _fresh(reqs[6]))], 48: [(3, _fresh(reqs[7]))]}
    mixed_c, mixed_l = _drive(sess, ev, 110)
    for r in reqs:
        sess = SlotSession(m, slots, 48, use_sampling=True, temp=2.0, top_k=3, top_p=0.0, cfg_coef=0.5)
        alone_c, alone_l = _drive(sess, {0: [(0, _fresh(r))]}, 50)
        assert torch.equal(mixed_c[r.id], alone_c[r.id]), f'request {r.id} ({OPTIONS[r.id]}): tokens differ from alone'
        assert torch.equal(mixed_l[r.id], alone_l[r.id]), f'request {r.id}: logits differ from alone'
        if slots == 4:   # teacher forcing runs one item, on the GEMM regime of up to 64 rows
            lg = m.teacher_forced_logits(_sequence(m, mixed_c[r.id].cpu()), r.cross, r.cfg_coef)[:, 0]
            assert torch.equal(mixed_l[r.id], lg), f'request {r.id}: logits differ from teacher forcing by ' \
                                                   f'{(mixed_l[r.id] - lg).abs().max():.3e}'
    if slots == 4:
        _check_generate(m, reqs, monkeypatch)
    print(f'slots={slots}: {len(reqs)} requests with mixed options bit-identical to each alone'
          + (', to teacher forcing and to generate' if slots == 4 else ''))


def _check_generate(m, reqs, monkeypatch):
    """generate draws its Philox key with torch.randint after the caller's seed; the session's requests take the key drawn
    the same way."""
    for r in reqs:
        torch.manual_seed(r.id)
        key = int(torch.randint(0, 2 ** 62, (1,)).item())
        sess = SlotSession(m, 4, 48)
        rr = _fresh(r)
        rr.seed = key
        c, _ = _drive(sess, {0: [(2, rr)]}, 50)
        monkeypatch.setenv('ACB_LM_PREFILL', '0')
        torch.manual_seed(r.id)
        want = m.generate(None if r.prompt is None else r.prompt.cuda(), [], num_samples=1, max_gen_len=r.max_gen_len,
                          use_sampling=r.use_sampling, temp=r.temp, top_k=r.top_k, top_p=r.top_p, cfg_coef=r.cfg_coef,
                          cross_attention_src=r.cross)
        monkeypatch.delenv('ACB_LM_PREFILL')
        assert torch.equal(c[r.id].cpu(), want.cpu()), f'request {r.id} ({OPTIONS[r.id]}): tokens differ from generate'


def test_cancel_mid_decode():
    cfg, sd, m = _model('lm_mini')
    reqs = _requests(cfg, sd)
    newcomer = _fresh(reqs[6])
    base = {0: [(0, _fresh(reqs[0])), (1, _fresh(reqs[1])), (2, _fresh(reqs[3])), (3, _fresh(reqs[5]))]}
    ref_c, ref_l = _drive(SlotSession(m, 4, 48), base, 50)
    # the same, with request 3 (top-p, slot 2) cancelled after 10 steps and the newcomer admitted into its slot
    ev = {0: [(s, _fresh(r)) for s, r in base[0]], 10: [(2, newcomer)]}
    got_c, got_l = _drive(SlotSession(m, 4, 48), ev, 60, cancels={10: [2]})
    assert 3 not in got_c and got_l[3].shape[0] == 10
    assert torch.equal(got_l[3], ref_l[3][:10]), 'the cancelled request differs before its cancel'
    for i in (0, 1, 5):
        assert torch.equal(got_c[i], ref_c[i]) and torch.equal(got_l[i], ref_l[i]), f'request {i} changed by the cancel'
    alone_c, alone_l = _drive(SlotSession(m, 4, 48), {0: [(0, _fresh(reqs[6]))]}, 50)
    assert torch.equal(got_c[6], alone_c[6]) and torch.equal(got_l[6], alone_l[6]), 'the newcomer differs from alone'


# ----------------------------------------------------------------------------- public path, streamed

PUBLIC_OPTIONS = [dict(), dict(use_sampling=False), dict(top_k=5, temperature=0.7), dict(top_p=0.9, top_k=0),
                  dict(temperature=1.3, cfg_coef=7.0), dict(cfg_coef=1.0)]


def _public_check(mg, requests, monkeypatch, victim):
    """requests: [(description, duration, prompt, options)].  The streamed session gets them all plus `victim`, cancelled
    after its first event; the non-streamed one gets them without it."""
    def submit(gen, items):
        ids = {}
        for i, (desc, dur, prompt, opts) in items:
            torch.manual_seed(1000 + i)
            ids[gen.submit(desc, duration=dur, prompt=prompt, prompt_sample_rate=None if prompt is None else mg.sample_rate,
                           **opts)] = i
        return ids

    items = list(enumerate(requests))
    gen = mg.continuous(slots=4, return_tokens=True)
    ids = submit(gen, items)
    whole = {ids[rid]: (wav, tok) for rid, wav, tok in gen.run()}

    gen = mg.continuous(slots=4, chunk_duration=0.2, return_tokens=True)
    ids = submit(gen, items[:2] + [(len(requests), victim)] + items[2:])
    victim_id = [rid for rid, i in ids.items() if i == len(requests)][0]
    pieces = {i: [] for i in ids.values()}
    finals, cancelled, first_at, polls = set(), False, {}, 0
    while gen.pending:
        for rid, piece, tok, final in gen.poll():
            i = ids[rid]
            assert i not in finals, 'an event after the final one'
            assert not (cancelled and rid == victim_id), 'an event after the cancel'
            pieces[i].append((piece, tok))
            first_at.setdefault(i, polls)
            if final:
                finals.add(i)
        polls += 1
        if not cancelled and len(requests) in first_at:
            assert gen.cancel(victim_id) and not gen.cancel(victim_id)
            cancelled = True
    assert cancelled and len(requests) not in finals
    assert finals == set(range(len(requests)))
    worst = 0.0
    for i, (desc, dur, prompt, opts) in items:
        wav = torch.cat([p for p, _ in pieces[i]], dim=-1)
        tok = torch.cat([t for _, t in pieces[i]], dim=-1)
        assert torch.equal(tok, whole[i][1]), f'request {i}: streamed tokens differ from the session'
        assert torch.equal(wav, whole[i][0]), f'request {i}: streamed audio differs from the session by ' \
                                              f'{(wav - whole[i][0]).abs().max():.3e}'
        params = dict(use_sampling=True, top_k=250, top_p=0.0, temperature=1.0, cfg_coef=3.0)
        params.update(opts)
        mg.set_generation_params(duration=dur, **params)
        monkeypatch.setenv('ACB_LM_PREFILL', '0')
        torch.manual_seed(1000 + i)
        if prompt is None:
            gwav, gtok = mg.generate([desc], return_tokens=True)
        else:
            gwav, gtok = mg.generate_continuation(prompt, mg.sample_rate, [desc], return_tokens=True)
        monkeypatch.delenv('ACB_LM_PREFILL')
        assert torch.equal(tok, gtok), f'request {i} ({opts}): tokens differ from generate'
        assert wav.shape == gwav.shape
        worst = max(worst, (wav - gwav).abs().max().item())
    mg.set_generation_params()
    print(f'{mg.name}: {len(requests)} streamed requests in {polls} polls, first pieces at polls {sorted(first_at.items())}, '
          f'max |pieces - generate| {worst:.2e}')
    assert worst <= WAV_TOL


def test_musicgen_streamed_session(monkeypatch):
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/small')
    prompt = H.audio_input(dict(sample_rate=32000, channels=1), 1, 6400, 3)
    descs = [('a tune', 0.5, None), ('piano', 0.8, prompt[0]), (None, 0.3, None), ('drums and bass', 1.0, None),
             ('b b', 0.62, None), ('strings', 0.9, None)]
    reqs = [d + (o,) for d, o in zip(descs, PUBLIC_OPTIONS)]
    _public_check(mg, reqs, monkeypatch, ('victim', 1.0, None, dict(top_p=0.9)))


def test_stereo_streamed_session(monkeypatch):
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/stereo-small')
    descs = [('a tune', 0.5, None), ('drums', 0.7, None), (None, 0.3, None), ('strings', 0.44, None)]
    reqs = [d + (o,) for d, o in zip(descs, PUBLIC_OPTIONS[1:])]
    _public_check(mg, reqs, monkeypatch, ('victim', 0.8, None, dict()))


def _audiogen():
    from audiocraft_b200.encodec import EncodecModel
    from audiocraft_b200.loaders import load_lm_model
    from audiocraft_b200.musicgen import AudioGen
    lm = load_lm_model('synthetic/lm_mini')
    ccfg = dict(synth.ENCODEC_CONFIGS['encodec_16k'], bins=lm.card)
    return AudioGen('debug', EncodecModel(synth.synth_encodec_state_dict(ccfg, 1), ccfg), lm, max_duration=10)


def test_audiogen_streamed_session(monkeypatch):
    ag = _audiogen()
    descs = [('dog barking', 0.5, None), ('rain', 1.0, None), (None, 0.1, None), ('wind in the trees', 0.7, None),
             ('car', 0.3, None), ('door', 0.96, None)]
    reqs = [d + (o,) for d, o in zip(descs, PUBLIC_OPTIONS)]
    _public_check(ag, reqs, monkeypatch, ('victim', 0.9, None, dict(cfg_coef=7.0)))


def test_groupnorm_codec_refuses_streamed_session():
    ag = _audiogen()
    gn = copy.copy(ag.compression_model)
    gn.cfg = dict(gn.cfg, norm='time_group_norm')
    ag.compression_model = gn
    session = ag.lm._session
    with pytest.raises(NotImplementedError, match='GroupNorm'):
        ag.continuous(slots=4, chunk_duration=0.2)
    assert ag.lm._session is session, 'a session was made before the refusal'
