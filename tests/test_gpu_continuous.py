"""GPU: continuous batching (slot mode of the decode step, `batching.SlotSession`, `BaseGenModel.continuous`).

* Inside a session, at capacity 4 (8 rows, lm_gemm_kernel) and 40 (80 rows, the wide GEMM): a request's tokens and per-step
  CFG-mixed logits are bit-identical alone, in another slot, among requests admitted at other steps with other text lengths,
  durations and prompts, and in a slot reused after another request retired from it.
* Against `LMModel.generate` of each item alone, greedy, on lm_mini, lm_tiny, rope, sin_rope and stereo configurations:
  descriptions of different lengths, unconditional requests, continuation prompts, durations from 2 frames to the session's
  maximum.  Tokens equal `generate` with the prompt fed one column per step (ACB_LM_PREFILL=0, what a session does); against
  the default prefilled `generate` a difference must start at an argmax near-tie (the rule of tests/test_gpu_lm.py).
* A 1-token condition next to a 60-token one: tokens and logits equal each generated alone.
* The public path: `continuous(slots=4)` with 10 sampled requests on synthetic MusicGen-small, and on an AudioGen model:
  tokens equal `generate` of the request alone after the same seed, waveforms within the EnCodec tolerance.
"""
import pytest
import torch

from audiocraft_b200 import synth
from audiocraft_b200.batching import ContinuousScheduler, Request, SlotSession
from tests import helpers as H

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4
NEAR_TIE = 5e-2


def _model(name, pe='sin', wseed=5):
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    cfg['positional_embedding'] = pe
    sd = synth.synth_lm_state_dict(cfg, seed=wseed)
    return cfg, sd, LMModel(sd, cfg, None, None)


def _cross(cfg, sd, T, seed):
    """[2, T, d]: a seeded condition row and its null (zero) row, like the condition provider's [cond; null]."""
    return H.lm_condition(cfg, sd, 1, T, seed)[2]


def _prompt(cfg, T0, seed):
    if T0 == 0:
        return None
    return torch.randint(0, cfg['card'], (1, cfg['n_q'], T0), generator=torch.Generator().manual_seed(seed))


def _drive(sess, events, n_total):
    """Run n_total steps through SlotSession.step_logits, admitting events[step] = [(slot, req)] before each step.
    Returns ({id: codes}, {id: logits [n_steps, K, card]})."""
    logs, active, codes = {}, {}, {}
    for t in range(n_total):
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


# ----------------------------------------------------------------------------- bit-identity inside a session

@pytest.mark.parametrize('slots', [4, 40])
@pytest.mark.parametrize('pe', ['sin', 'rope'])
def test_request_is_independent_of_slot_neighbours_and_history(slots, pe):
    cfg, sd, m = _model('lm_mini', pe)

    def target():
        return Request(37, _cross(cfg, sd, 9, 1), _prompt(cfg, 5, 2), seed=123, id=0)

    def others():
        return [Request(12, _cross(cfg, sd, 3, 3), None, seed=7, id=1),
                Request(50, _cross(cfg, sd, 30, 4), _prompt(cfg, 11, 5), seed=8, id=2),
                Request(2, torch.zeros(2, 1, cfg['dim']), None, seed=9, id=3),
                Request(20, _cross(cfg, sd, 60, 6), None, seed=10, id=4)]

    for sampling in (False, True):
        sess = SlotSession(m, slots, 64, use_sampling=sampling, top_k=20, temp=1.1)
        alone_c, alone_l = _drive(sess, {0: [(0, target())]}, 40)
        sess = SlotSession(m, slots, 64, use_sampling=sampling, top_k=20, temp=1.1)
        other_c, other_l = _drive(sess, {0: [(slots - 1, target())]}, 40)
        o = others()
        sess = SlotSession(m, slots, 64, use_sampling=sampling, top_k=20, temp=1.1)
        # slot 1 first hosts request 3 (2 frames: retires after 5 steps), then the target at step 6; the others come and go
        crowd_c, crowd_l = _drive(sess, {0: [(1, o[2]), (0, o[0])], 2: [(2, o[1])], 6: [(1, target())],
                                         20: [(0, o[3])], 30: [(3, Request(2, torch.zeros(2, 1, cfg['dim']), None, 9, id=5))]},
                                   90)
        assert torch.isfinite(alone_l[0]).all()
        for name, c, lg in (('other slot', other_c, other_l), ('crowded, reused slot', crowd_c, crowd_l)):
            assert torch.equal(c[0], alone_c[0]), f'{name}: tokens differ'
            assert torch.equal(lg[0], alone_l[0]), f'{name}: logits differ by {(lg[0] - alone_l[0]).abs().max():.3e}'
        # a slot reused after a request with a longer condition, a prompt and another length: as fresh
        sess = SlotSession(m, slots, 64, use_sampling=sampling, top_k=20, temp=1.1)
        reuse_c, reuse_l = _drive(sess, {0: [(0, others()[1])], 60: [(0, target())]}, 100)
        assert torch.equal(reuse_c[0], alone_c[0]) and torch.equal(reuse_l[0], alone_l[0])
        print(f'slots={slots} {pe} sampling={sampling}: alone / other slot / crowded / reused slot bit-identical')


# ----------------------------------------------------------------------------- parity with generate

def _generate_alone(m, req, monkeypatch, prefill):
    monkeypatch.setenv('ACB_LM_PREFILL', '1' if prefill else '0')
    out = m.generate(None if req.prompt is None else req.prompt.cuda(), [], num_samples=1, max_gen_len=req.max_gen_len,
                     use_sampling=False, cross_attention_src=req.cross)
    monkeypatch.delenv('ACB_LM_PREFILL')
    return out.cpu()


def _sequence(m, codes):
    """codes [1, K, T] -> the delay-pattern sequence [1, K, S] generate builds from them."""
    return m.pattern_provider.get_pattern(codes.shape[-1]).build_pattern_sequence(codes, m.special_token_id)[0]


def _near_tie(m, req, got, want):
    """The first sequence step where got and want differ must be an argmax near-tie of the logits along got's path."""
    seq = _sequence(m, got)
    lg = m.teacher_forced_logits(seq, req.cross, m.cfg_coef).cpu()   # [S - 1, 1, K, card]
    wseq = _sequence(m, want)
    step = int((seq != wseq).any(0).any(0).nonzero()[0])
    top2 = lg[step - 1].topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).min().item()
    assert margin < NEAR_TIE, f'differs at sequence step {step} although the argmax margin is {margin:.3e}'
    return margin


def _mixed_requests(cfg, sd, max_len, seed):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(11):
        T = [1, 3, 16, 60][i % 4]
        n = [2, max_len, 9, 23, 31, 5][i % 6]
        cross = torch.zeros(2, T, cfg['dim']) if i % 5 == 4 else _cross(cfg, sd, T, 100 + i)   # unconditional every 5th
        T0 = [0, 0, 4, 1, 7][i % 5] if n > 8 else 0
        reqs.append(Request(n, cross, _prompt(cfg, T0, 200 + i), seed=int(torch.randint(0, 2 ** 62, (1,), generator=g)), id=i))
    return reqs


@pytest.mark.parametrize('name,pe', [('lm_mini', 'sin'), ('lm_tiny', 'sin'), ('lm_mini', 'rope'), ('lm_mini', 'sin_rope'),
                                     ('lm_mini_stereo', 'sin')])
def test_greedy_session_equals_generate_alone(monkeypatch, name, pe):
    cfg, sd, m = _model(name, pe)
    max_len = 40
    reqs = _mixed_requests(cfg, sd, max_len, seed=3)
    sched = ContinuousScheduler(SlotSession(m, 4, max_len, use_sampling=False), 4)
    for r in reqs:
        sched.submit(r)
    got = {}
    while sched.pending:
        for r, codes in sched.poll():
            got[r.id] = codes.cpu()
    assert sorted(got) == [r.id for r in reqs]
    margins = []
    for r in reqs:
        assert got[r.id].shape == (1, cfg['n_q'], r.max_gen_len)
        if r.prompt is not None:
            assert torch.equal(got[r.id][..., :r.prompt.shape[-1]], r.prompt), 'the prompt must come back unchanged'
        assert torch.equal(got[r.id], _generate_alone(m, r, monkeypatch, prefill=False)), f'request {r.id}'
        want = _generate_alone(m, r, monkeypatch, prefill=True)
        if not torch.equal(got[r.id], want):
            margins.append(_near_tie(m, r, got[r.id], want))
    print(f'{name} {pe}: {len(reqs)} requests equal generate alone; occupancy {sched.occupancy:.2f}, '
          f'{len(margins)} near-ties against the prefilled path {margins}')


def test_short_and_long_condition_side_by_side():
    """Each slot attends over exactly its own text length: a 1-token condition next to a 60-token one gives the tokens and
    logits of each generated alone.  (With one text length shared by the slots, the short one attends to 59 more keys.)"""
    cfg, sd, m = _model('lm_mini')
    short, long_ = _cross(cfg, sd, 1, 11), _cross(cfg, sd, 60, 12)
    sess = SlotSession(m, 4, 32, use_sampling=False)
    codes, logits = _drive(sess, {0: [(0, Request(24, long_, id=0)), (1, Request(24, short, id=1))]}, 30)
    for i, cross in ((0, long_), (1, short)):
        alone = m.generate(None, [], num_samples=1, max_gen_len=24, use_sampling=False, cross_attention_src=cross).cpu()
        assert torch.equal(codes[i].cpu(), alone), f'request {i}: tokens differ from generate alone'
        lg = m.teacher_forced_logits(_sequence(m, codes[i].cpu()), cross, m.cfg_coef)[:, 0]
        assert torch.equal(logits[i], lg), f'request {i}: logits differ by {(logits[i] - lg).abs().max():.3e}'


# ----------------------------------------------------------------------------- public path

def _public_check(mg, requests, monkeypatch):
    gen = mg.continuous(slots=4, return_tokens=True)
    ids = {}
    for i, (desc, dur, prompt) in enumerate(requests):
        torch.manual_seed(1000 + i)
        ids[gen.submit(desc, duration=dur, prompt=prompt, prompt_sample_rate=None if prompt is None else mg.sample_rate)] = i
    got = {}
    for rid, wav, tok in gen.run():
        got[ids[rid]] = (wav, tok)
    assert sorted(got) == list(range(len(requests)))
    worst = 0.0
    for i, (desc, dur, prompt) in enumerate(requests):
        mg.set_generation_params(duration=dur)
        monkeypatch.setenv('ACB_LM_PREFILL', '0')   # a session feeds a prompt one column per step
        torch.manual_seed(1000 + i)
        if prompt is None:
            wav, tok = mg.generate([desc], return_tokens=True)
        else:
            wav, tok = mg.generate_continuation(prompt, mg.sample_rate, [desc], return_tokens=True)
        monkeypatch.delenv('ACB_LM_PREFILL')
        gw, gt = got[i]
        assert torch.equal(gt, tok), f'request {i}: tokens differ'
        assert gw.shape == wav.shape, (i, gw.shape, wav.shape)
        worst = max(worst, (gw - wav).abs().max().item())
    print(f'{mg.name}: {len(requests)} requests, occupancy {gen.occupancy:.2f}, max |wav - generate| {worst:.2e}')
    assert worst <= WAV_TOL


def test_musicgen_continuous_equals_generate(monkeypatch):
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/small')
    prompt = H.audio_input(dict(sample_rate=32000, channels=1), 1, 6400, 3)
    reqs = [('a tune', 0.5, None), ('drums and a long description of many words here', 1.0, None), (None, 0.3, None),
            ('x', 0.04, None), ('piano', 0.8, prompt[0]), ('a', 0.5, None), ('b b', 0.62, None), (None, 1.0, None),
            ('c', 0.2, None), ('strings', 0.9, None)]
    _public_check(mg, reqs, monkeypatch)
    with pytest.raises(NotImplementedError):
        mg.continuous(slots=2).submit('too long', duration=mg.max_duration + 1)


def test_audiogen_continuous_equals_generate(monkeypatch):
    from audiocraft_b200.encodec import EncodecModel
    from audiocraft_b200.loaders import load_lm_model
    from audiocraft_b200.musicgen import AudioGen
    lm = load_lm_model('synthetic/lm_mini')
    ccfg = dict(synth.ENCODEC_CONFIGS['encodec_16k'], bins=lm.card)
    ag = AudioGen('debug', EncodecModel(synth.synth_encodec_state_dict(ccfg, 1), ccfg), lm, max_duration=10)
    reqs = [('dog barking', 0.5, None), ('rain', 1.0, None), (None, 0.1, None), ('wind in the trees', 0.7, None),
            ('car', 0.3, None), ('door', 0.96, None)]
    _public_check(ag, reqs, monkeypatch)
