"""GPU: continuous batching of models with a condition prefix (the `prepend` fuser, MusicGen-melody): each request's prefix
is prefilled into its own slot at admission (acb_lm_admit_prefix) and the slot runs column t at cache position P + t.

* Inside a session, at 4 slots (8 rows) and 40 slots (80 rows, the wide GEMM), sin and rope, with and without cross
  attention: a request with a 37-position prefix gives bit-identical tokens and per-step CFG-mixed logits alone, in another
  slot, among requests with 1-, 60- and 0-position prefixes admitted at other steps, and in a slot reused after a request
  with a longer prefix.
* Admission K/V: the slot's cache rows hold bit for bit what `LMModel.generate(prefix=...)` of the request alone writes, and
  no other slot's rows change.
* Greedy parity with `generate` alone: equal tokens at 4 slots (prompts fed one column per step, ACB_LM_PREFILL=0); at 40
  slots a difference must start at an argmax near-tie.
* The public path on the lm_mini_melody golden model and on a stereo-melody one: `continuous(slots=4)` equals
  `generate_with_chroma` / `generate` / `generate_continuation` alone after the same seed; against the reference's golden
  tokens and logits; streamed pieces; refused admissions that leave the session unchanged.
"""
import ctypes as C

import pytest
import torch

from audiocraft_b200 import _lib, synth
from audiocraft_b200.batching import ContinuousScheduler, Request, SlotSession
from audiocraft_b200.conditioners import ConditionFuser
from tests import helpers as H
from tests import melody_golden as MG
from tests.prefix_oracle import PrefixLMOracle
from tests.test_gpu_continuous import _drive, _sequence

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4
NEAR_TIE = 5e-2
MAX_PREFIX = 64


def _model(pe='sin', cross=True, wseed=5):
    """lm_mini with a `prepend` fuser: [self_wav] prefix + description by cross attention, or [self_wav, description] prefix
    and no cross attention (the released melody layout)."""
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config('lm_mini')
    cfg['positional_embedding'] = pe
    cfg['cross_attention'] = cross
    sd = synth.synth_lm_state_dict(cfg, seed=wseed)
    fuser = ConditionFuser({'prepend': ['self_wav'], 'cross': ['description']} if cross else
                           {'prepend': ['self_wav', 'description']})
    return cfg, sd, LMModel(sd, cfg, None, fuser)


def _prefix(cfg, P, seed):
    """[2, P, d]: distinct cond and null rows, magnitudes like output_proj outputs."""
    return torch.randn(2, P, cfg['dim'], generator=torch.Generator().manual_seed(seed)) * 0.5


def _cross(cfg, sd, T, seed):
    return H.lm_condition(cfg, sd, 1, T, seed)[2] if cfg['cross_attention'] else None


def _prompt(cfg, T0, seed):
    if T0 == 0:
        return None
    return torch.randint(0, cfg['card'], (1, cfg['n_q'], T0), generator=torch.Generator().manual_seed(seed))


def _req(cfg, sd, n, P, T, T0, seed, rid, pseed):
    return Request(n, _cross(cfg, sd, T, pseed), _prompt(cfg, T0, pseed + 1), seed=seed, id=rid,
                   prefix=_prefix(cfg, P, pseed + 2))


def _session(m, slots, sampling=True):
    return SlotSession(m, slots, 64, use_sampling=sampling, top_k=20, temp=1.1, max_prefix=MAX_PREFIX)


# ----------------------------------------------------------------------------- bit-identity inside a session

@pytest.mark.parametrize('cross', [True, False])
@pytest.mark.parametrize('pe', ['sin', 'rope'])
@pytest.mark.parametrize('slots', [4, 40])
def test_prefix_request_is_independent_of_slot_neighbours_and_history(slots, pe, cross):
    cfg, sd, m = _model(pe, cross)

    def target():
        return _req(cfg, sd, 30, 37, 9, 5, 123, 0, 1)

    def others():
        return [_req(cfg, sd, 12, 1, 3, 0, 7, 1, 10), _req(cfg, sd, 40, 60, 30, 11, 8, 2, 20),
                _req(cfg, sd, 2, 0, 1, 0, 9, 3, 30), _req(cfg, sd, 20, 60, 60, 0, 10, 4, 40)]

    for sampling in (False, True):
        alone_c, alone_l = _drive(_session(m, slots, sampling), {0: [(0, target())]}, 40)
        other_c, other_l = _drive(_session(m, slots, sampling), {0: [(slots - 1, target())]}, 40)
        o = others()
        # slot 1 first hosts request 3 (P = 0, 2 frames: retires after 5 steps), then the target at step 6
        crowd_c, crowd_l = _drive(_session(m, slots, sampling),
                                  {0: [(1, o[2]), (0, o[0])], 2: [(2, o[1])], 6: [(1, target())], 20: [(0, o[3])]}, 90)
        # slot 0 reused after a request with a longer prefix (60), a longer condition, a prompt and another length
        reuse_c, reuse_l = _drive(_session(m, slots, sampling), {0: [(0, others()[1])], 50: [(0, target())]}, 90)
        assert torch.isfinite(alone_l[0]).all()
        for name, c, lg in (('other slot', other_c, other_l), ('crowded', crowd_c, crowd_l), ('reused slot', reuse_c, reuse_l)):
            assert torch.equal(c[0], alone_c[0]), f'{name}: tokens differ'
            assert torch.equal(lg[0], alone_l[0]), f'{name}: logits differ by {(lg[0] - alone_l[0]).abs().max():.3e}'
        print(f'slots={slots} {pe} cross={cross} sampling={sampling}: alone / other slot / crowded / reused bit-identical')


# ----------------------------------------------------------------------------- admission K/V

@pytest.mark.parametrize('cross', [True, False])
def test_admission_kv_equals_generate_alone(cross):
    cfg, sd, m = _model('sin', cross)
    slots, s, P = 4, 2, 37
    sess = _session(m, slots)
    for k in (0, 1, 3):   # the other slots hold requests with prefixes of their own
        sess.admit(k, _req(cfg, sd, 20, [5, 60, 33][k % 3], 7, 0, k, 10 + k, 50 + 10 * k))
    sess.steps(3)
    b = m._bufs
    before_k, before_v = b['k_cache'].clone(), b['v_cache'].clone()
    req = _req(cfg, sd, 30, P, 9, 0, 5, 9, 1)
    sess.admit(s, req)
    torch.cuda.synchronize()
    rows = [s, slots + s]
    got_k, got_v = b['k_cache'][:, rows, :, :P].clone(), b['v_cache'][:, rows, :, :P].clone()
    others = [r for r in range(b['k_cache'].shape[1]) if r not in rows]
    assert torch.equal(b['k_cache'][:, others], before_k[:, others]), "another slot's K rows changed"
    assert torch.equal(b['v_cache'][:, others], before_v[:, others]), "another slot's V rows changed"
    m.generate(None, [], num_samples=1, max_gen_len=30, use_sampling=False, cross_attention_src=req.cross, prefix=req.prefix)
    b = m._bufs
    assert torch.equal(got_k, b['k_cache'][:, :2, :, :P]), 'K of the admitted prefix differ from generate alone'
    assert torch.equal(got_v, b['v_cache'][:, :2, :, :P]), 'V of the admitted prefix differ from generate alone'


# ----------------------------------------------------------------------------- parity with generate

def _mixed(cfg, sd, max_len, seed):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(10):
        n = [2, max_len, 9, 23, 31][i % 5]
        T0 = [0, 4, 0, 7][i % 4] if n > 8 else 0
        reqs.append(_req(cfg, sd, n, [1, 37, 60, 13, 0, 64][i % 6], [1, 3, 16, 60][i % 4], T0,
                         int(torch.randint(0, 2 ** 62, (1,), generator=g)), i, 100 + 10 * i))
    return reqs


def _alone(m, r, monkeypatch):
    monkeypatch.setenv('ACB_LM_PREFILL', '0')   # a session feeds a prompt one column per step
    out = m.generate(None if r.prompt is None else r.prompt.cuda(), [], num_samples=1, max_gen_len=r.max_gen_len,
                     use_sampling=False, cross_attention_src=r.cross, prefix=r.prefix)
    monkeypatch.delenv('ACB_LM_PREFILL')
    return out.cpu()


@pytest.mark.parametrize('cross,pe', [(True, 'sin'), (False, 'rope'), (True, 'sin_rope')])
@pytest.mark.parametrize('slots', [4, 40])
def test_greedy_session_equals_generate_alone(monkeypatch, slots, cross, pe):
    cfg, sd, m = _model(pe, cross)
    reqs = _mixed(cfg, sd, 40, seed=3)
    sched = ContinuousScheduler(SlotSession(m, slots, 40, use_sampling=False, max_prefix=MAX_PREFIX), slots)
    for r in reqs:
        sched.submit(r)
    got = {}
    while sched.pending:
        for r, codes in sched.poll():
            got[r.id] = codes.cpu()
    margins = []
    for r in reqs:
        assert got[r.id].shape == (1, cfg['n_q'], r.max_gen_len)
        if r.prompt is not None:
            assert torch.equal(got[r.id][..., :r.prompt.shape[-1]], r.prompt)
        want = _alone(m, r, monkeypatch)
        if slots * 2 <= 64:
            assert torch.equal(got[r.id], want), f'request {r.id} (P = {r.prefix.shape[1]})'
        elif not torch.equal(got[r.id], want):   # the wide GEMM sums in another order: a difference starts at a near-tie
            seq = _sequence(m, got[r.id])
            lg = m.teacher_forced_logits(seq, r.cross, m.cfg_coef, prefix=r.prefix).cpu()
            step = int((seq != _sequence(m, want)).any(0).any(0).nonzero()[0])
            top2 = lg[step - 1].topk(2, dim=-1).values
            margin = (top2[..., 0] - top2[..., 1]).min().item()
            assert margin < NEAR_TIE, f'request {r.id}: differs at step {step} with argmax margin {margin:.3e}'
            margins.append(margin)
    print(f'slots={slots} cross={cross} {pe}: {len(reqs)} requests equal generate alone, near-ties {margins}')


# ----------------------------------------------------------------------------- refused admissions

def test_refused_admissions_leave_the_session_unchanged():
    cfg, sd, m = _model('sin', True)

    def run(refuse):
        sess = _session(m, 4)
        events = {0: [(0, _req(cfg, sd, 30, 37, 9, 0, 5, 0, 1))], 3: [(2, _req(cfg, sd, 12, 20, 4, 0, 6, 1, 2))]}
        logs, codes = {}, {}
        for t in range(45):
            for slot, req in events.get(t, []):
                sess.admit(slot, req)
                logs[req.id] = (slot, req, [])
            if refuse and t == 5:
                lm = m
                samp = C.byref(_lib.LMSampling(1, 1.0, 20, 0.0, 3.0, 0, 0, 0.0))
                cross = _cross(cfg, sd, 3, 9).cuda().contiguous()
                pre = _prefix(cfg, 8, 9).cuda()
                max_seq = lm._shape[1]
                for args, what in (((pre.data_ptr(), max_seq, 10), 'prefix + seq_len > max_seq'),
                                   ((None, 8, 10), 'null prefix'),
                                   ((pre.data_ptr(), -1, 10), 'negative prefix_len')):
                    rc = lm._lib.acb_lm_admit_prefix(lm._handle, 1, cross.data_ptr(), 3, args[0], args[1], args[2],
                                                     C.c_uint64(3), samp, _lib.stream())
                    assert rc != 0, what
                with pytest.raises(ValueError):
                    sess.admit(1, Request(10, cross.cpu(), None, seed=1, id=7))   # no prefix on a prefix model
                with pytest.raises(ValueError):
                    sess.admit(1, Request(10, cross.cpu(), None, seed=1, id=7, prefix=_prefix(cfg, MAX_PREFIX + 1, 1)))
            lg = sess.step_logits()
            for rid, (slot, req, lst) in logs.items():
                if rid not in codes:
                    lst.append(lg[slot].clone())
                    if len(lst) == req.meta['S'] - 1:
                        codes[rid] = sess.collect(slot, req)
        assert sorted(codes) == [0, 1]
        assert all(st != 1 for _, st in sess.status())
        return codes, {k: torch.stack(v[2]) for k, v in logs.items()}

    c0, l0 = run(False)
    c1, l1 = run(True)
    for k in c0:
        assert torch.equal(c0[k], c1[k]) and torch.equal(l0[k], l1[k]), f'request {k} changed after a refused admission'


# ----------------------------------------------------------------------------- public path

def _golden_musicgen(case='sin_matchlen'):
    from audiocraft_b200.loaders import load_compression_model
    from audiocraft_b200.lm import LMModel
    from audiocraft_b200.musicgen import MusicGen
    g = MG.golden()
    cfg = MG.config(g, case)
    sd = MG.weights(g, cfg)
    prov, fuser = MG.provider_and_fuser(g, case, cfg, sd)
    lm = LMModel(sd, cfg, prov, fuser, 'cuda')
    return g, cfg, sd, MusicGen('golden/lm_mini_melody', load_compression_model('synthetic/encodec_32k', 'cuda', 1), lm,
                                max_duration=30)


def _stereo_melody_musicgen():
    from audiocraft_b200.encodec import get_wrapped_compression_model
    from audiocraft_b200.loaders import _STEREO_WRAP, load_compression_model, load_lm_model
    from audiocraft_b200.musicgen import MusicGen
    lm = load_lm_model('synthetic/lm_mini_melody_stereo')
    cm = get_wrapped_compression_model(load_compression_model('synthetic/encodec_32k', 'cuda', 1), **_STEREO_WRAP)
    return MusicGen('synthetic/stereo-lm_mini_melody', cm, lm, max_duration=30)


def _melody(seconds, seed, channels=1):
    return H.audio_input(dict(sample_rate=32000, channels=channels), 1, int(32000 * seconds), seed)[0]


def _run_session(mg, reqs, chunk_duration=None):
    gen = mg.continuous(slots=4, return_tokens=True, chunk_duration=chunk_duration)
    ids = {}
    for i, (desc, dur, melody, prompt) in enumerate(reqs):
        torch.manual_seed(1000 + i)
        ids[gen.submit(desc, duration=dur, melody=melody, melody_sample_rate=None if melody is None else 32000,
                       prompt=prompt, prompt_sample_rate=None if prompt is None else mg.sample_rate)] = i
    got = {}
    if chunk_duration is None:
        for rid, wav, tok in gen.run():
            got[ids[rid]] = (wav, tok)
    else:
        pieces = {}
        for rid, piece, tok, final in gen.run():
            pieces.setdefault(ids[rid], []).append((piece, tok))
        for i, ps in pieces.items():
            got[i] = (torch.cat([p for p, _ in ps], -1), torch.cat([t for _, t in ps], -1))
    assert sorted(got) == list(range(len(reqs)))
    return got, gen.occupancy


def _public_check(mg, reqs, monkeypatch):
    got, occ = _run_session(mg, reqs)
    worst = 0.0
    for i, (desc, dur, melody, prompt) in enumerate(reqs):
        mg.set_generation_params(duration=dur, **{k: v for k, v in SAMPLING.items()})
        monkeypatch.setenv('ACB_LM_PREFILL', '0')
        torch.manual_seed(1000 + i)
        if melody is not None:
            wav, tok = mg.generate_with_chroma([desc], melody, 32000, return_tokens=True)
        elif prompt is not None:
            wav, tok = mg.generate_continuation(prompt, mg.sample_rate, [desc], return_tokens=True)
        else:
            wav, tok = mg.generate([desc], return_tokens=True)
        monkeypatch.delenv('ACB_LM_PREFILL')
        gw, gt = got[i]
        assert torch.equal(gt, tok), f'request {i}: tokens differ'
        assert gw.shape == wav.shape, (i, gw.shape, wav.shape)
        worst = max(worst, (gw - wav).abs().max().item())
    print(f'{mg.name}: {len(reqs)} requests, occupancy {occ:.2f}, max |wav - alone| {worst:.2e}')
    assert worst <= WAV_TOL
    return got


SAMPLING = dict(use_sampling=True, top_k=50, temperature=1.0)


def _public_requests(channels, descs):
    prompt = H.audio_input(dict(sample_rate=32000, channels=channels), 1, 6400, 3)[0]
    d0, d1 = descs
    return [(d0, 0.5, _melody(0.8, 1, channels), None), (d1, 0.3, None, None), (None, 0.4, _melody(2.0, 2, channels), None),
            (d1, 0.06, _melody(0.3, 3), None), (None, 0.5, None, None), (d0, 0.8, None, prompt),
            (d1, 0.62, _melody(1.1, 4, channels), None), (d0, 0.2, None, None), (None, 0.7, None, prompt),
            (d0, 0.9, _melody(0.5, 5, channels), None)]


def test_melody_continuous_equals_generate_alone(monkeypatch):
    g, cfg, sd, mg = _golden_musicgen()
    mg.set_generation_params(**SAMPLING)
    reqs = _public_requests(1, ('d0', 'd1'))
    got = _public_check(mg, reqs, monkeypatch)
    # streaming: each melody request's pieces, concatenated, are its waveform without chunk_duration
    mg.set_generation_params(**SAMPLING)
    streamed, _ = _run_session(mg, reqs, chunk_duration=0.2)
    for i in got:
        assert torch.equal(streamed[i][1], got[i][1]), f'request {i}: streamed tokens differ'
        torch.testing.assert_close(streamed[i][0], got[i][0], rtol=0, atol=1e-5)


def test_stereo_melody_continuous_equals_generate_alone(monkeypatch):
    mg = _stereo_melody_musicgen()
    assert mg.lm.n_q == 8
    mg.set_generation_params(**SAMPLING)
    _public_check(mg, _public_requests(2, ('a tune', 'drums and a long description of many words')), monkeypatch)


def test_session_matches_reference_golden():
    """The reference's MusicGen-melody golden (tests/golden/make_golden_melody.py): a slot teacher-forced on the golden's
    sequence (its known tokens are kept) gives CFG logits within 6e-2 of the reference's, and greedy session tokens are the
    reference's outside argmax near-ties of the fp16-emulating oracle."""
    case = 'sin_matchlen'
    g, cfg, sd, mg = _golden_musicgen(case)
    c = g['cases'][case]
    B, T = g['batch'], g['T']
    _, _, prefix = MG.repo_conditions(g, case, cfg, sd)
    lm = mg.lm
    seq = MG.teacher_sequence(g, cfg)
    sess = SlotSession(lm, 4, T, use_sampling=False, max_prefix=prefix.shape[1])
    reqs = [Request(T, None, None, seed=i, id=i, prefix=prefix[[i, B + i]]) for i in range(B)]
    for i, r in enumerate(reqs):
        sess.admit(i + 1, r)
        lm._bufs['seq'][i + 1, :, :seq.shape[-1]] = seq[i].cuda()   # known tokens stay: the slot is teacher-forced
    logits = [[] for _ in range(B)]
    for _ in range(seq.shape[-1] - 1):
        lg = sess.step_logits()
        for i in range(B):
            logits[i].append(lg[i + 1].cpu())
    lg = torch.stack([torch.stack(x) for x in logits], 1)   # [S - 1, B, K, card]
    err = (lg[..., c['logits_idx']] - c['logits']).abs().max().item()
    print(f'session logits vs the reference golden: max |diff| {err:.3e}')
    torch.testing.assert_close(lg[..., c['logits_idx']], c['logits'], rtol=6e-2, atol=6e-2)
    # greedy
    sess = SlotSession(lm, 4, T, use_sampling=False, max_prefix=prefix.shape[1])
    codes, _ = _drive(sess, {0: [(i, Request(T, None, None, seed=i, id=i, prefix=prefix[[i, B + i]])) for i in range(B)]},
                      T + 10)
    got = torch.cat([codes[i].cpu() for i in range(B)])
    if not torch.equal(got, c['greedy']):
        rec = []
        PrefixLMOracle(sd, cfg, half_gemm=True, prefix=prefix).generate(None, None, B, T, use_sampling=False,
                                                                         cfg_coef=cfg['cfg_coef'], record_logits=rec)
        top2 = torch.stack(rec).topk(2, dim=-1).values
        margin = (top2[..., 0] - top2[..., 1]).min().item()
        assert margin < NEAR_TIE, f'greedy session tokens differ from the reference although the margins are clear ({margin:.3e})'
        pytest.skip(f'greedy path hits an argmax near-tie (min margin {margin:.3e})')
