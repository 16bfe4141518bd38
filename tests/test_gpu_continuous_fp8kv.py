"""FP8 self-attention KV pool (SlotSession(kv_dtype='fp8'), continuous(kv_cache_dtype='fp8')) on the H100.

Kernel checks use the probe LM of tests/test_gpu_decode_f64.py (every out-projection and linear2 zero, every norm a copy of
out_norm, so h16 is the input of every layer's QKV GEMM) with one more change: every layer's self-attention in-projection is
the same signed power-of-two permutation, with the K rows equal to the Q rows.  Each fp32 q, k and v sum then has one non-zero
product and is exact, the K of every layer equals q before rotary positions, and under rotary positions the rotated K is
bit for bit the rotated q the step leaves in q32 (the same rope_rotate on the same inputs).  So the codes and scales the
step writes are compared bit for bit with tests/test_continuous_fp8kv_host.quant_e4m3 of values the CPU knows exactly:
K from q32 (after rotary positions), V from h16.  Before a step every code (0x7F, NaN in e4m3) and scale (NaN) the step must
not read is poisoned; the step must change exactly position n - 1 of each active row in every layer, and the attention
output must lie within the float64 bound on code x scale (fp8_attn64)."""
import math

import pytest
import torch

from audiocraft_b200 import _lib
from audiocraft_b200.batching import PagePool, Request, SlotSession, kv_page_bytes
from tests import test_gpu_continuous_melody as M
from tests.test_continuous_fp8kv_host import dequant, fp8_attn64, quant_e4m3
from tests.test_gpu_continuous_prefill import _small, _text_requests, _melody_requests
from tests.test_gpu_decode_f64 import _nan_equal
from tests.test_gpu_kernels_f64 import _synth, check, probe_state_dict

pytestmark = pytest.mark.gpu

PAGE = _lib.ACB_LM_KV_PAGE
POISON = 0x7F


def _probe_fp8(name, pe, cross, prefix=False, seed=7):
    from audiocraft_b200.conditioners import ConditionFuser
    from audiocraft_b200.lm import LMModel
    cfg0, sd0 = _synth(name, (), cross, seed)
    cfg = dict(cfg0, positional_embedding=pe)
    sd = probe_state_dict(cfg, sd0, ('self_attn.out_proj.weight', 'cross_attention.out_proj.weight', 'linear2.weight'), True)
    d = cfg['dim']
    g = torch.Generator().manual_seed(seed)
    w = torch.zeros(3 * d, d)
    pq, pv = torch.randperm(d, generator=g), torch.randperm(d, generator=g)
    sq = (2.0 ** torch.randint(-2, 3, (d,), generator=g)) * (torch.randint(0, 2, (d,), generator=g) * 2 - 1)
    sv = (2.0 ** torch.randint(-2, 3, (d,), generator=g)) * (torch.randint(0, 2, (d,), generator=g) * 2 - 1)
    w[torch.arange(d), pq] = sq
    w[d + torch.arange(d), pq] = sq
    w[2 * d + torch.arange(d), pv] = sv
    for li in range(cfg['num_layers']):
        sd[f'transformer.layers.{li}.self_attn.in_proj_weight'] = w.clone()
        if cross:
            p = f'transformer.layers.{li}.cross_attention.in_proj_weight'
            sd[p] = sd[p].clone()
            sd[p][:d] = torch.eye(d)
    fuser = ConditionFuser({'prepend': ['self_wav', 'description']}) if prefix else None
    return cfg, LMModel(sd, cfg, None, fuser), w


def _locs(sess, rows_pos):
    """[(row, pos, page, offset)] for rows_pos [(row, pos)]."""
    table = sess.page_table.cpu()
    return [(r, p, int(table[r, p // PAGE]), p % PAGE) for r, p in rows_pos]


def _poison(sess, keep):
    """Poison every code and scale except the (page, offset) pairs in `keep` (positions the next step may read)."""
    k8, v8 = sess.k_pool.view(torch.uint8), sess.v_pool.view(torch.uint8)
    mask = torch.ones(sess.k_scale.shape[1:2] + sess.k_scale.shape[3:], dtype=torch.bool)   # [n_pages, PAGE]
    for pg, off in keep:
        mask[pg, off] = False
    mask = mask.cuda()
    for c in (k8, v8):
        c.masked_fill_(mask[None, :, None, :, None], POISON)
    for s in (sess.k_scale, sess.v_scale):
        s.masked_fill_(mask[None, :, None, :], float('nan'))


def _snapshot(sess):
    return (sess.k_pool.view(torch.uint8).clone(), sess.v_pool.view(torch.uint8).clone(), sess.k_scale.clone(),
            sess.v_scale.clone())


def _check_written(sess, before, locs, tag):
    """Exactly the (page, offset) pairs in locs changed, in every layer, head, code and scale."""
    now = _snapshot(sess)
    for i, nm in enumerate(('k codes', 'v codes', 'k scales', 'v scales')):
        changed = now[i] != before[i] if i < 2 else ~_nan_equal(now[i], before[i])
        want = torch.zeros_like(changed)
        for _, _, pg, off in locs:
            want[:, pg, :, off] = True
        # a written value may equal the poison only for scales (never NaN) or a code that happens to be 0x7F (NaN: never)
        assert torch.equal(changed, want), f'{tag}: {nm} changed outside position n - 1 of the active rows'


def _check_codes(sess, cfg, w, h16, q32, locs, tag):
    """Codes and scales at locs (rows of h16 / q32 in the same order) are quant_e4m3 of the exact K / V in every layer."""
    d, Hn = cfg['dim'], cfg['num_heads']
    R = len(locs)
    rope = cfg['positional_embedding'] != 'sin'
    x = h16.float().cpu()
    k_exact = q32.float().cpu() if rope else x @ w[d:2 * d].t()      # exact: one non-zero product per sum
    if not rope:
        assert torch.equal(k_exact, q32.float().cpu()), f'{tag}: q32 is not the exact q'
    v_exact = x @ w[2 * d:].t()
    kc, ks = quant_e4m3(k_exact.view(R, Hn, 64))
    vc, vs = quant_e4m3(v_exact.view(R, Hn, 64))
    pg = torch.tensor([l[2] for l in locs]).cuda()
    off = torch.tensor([l[3] for l in locs]).cuda()
    for layer in range(cfg['num_layers']):
        for nm, pool, sc, wc, ws in (('k', sess.k_pool, sess.k_scale, kc, ks), ('v', sess.v_pool, sess.v_scale, vc, vs)):
            got_c = pool[layer][pg, :, off].view(torch.uint8).cpu()
            got_s = sc[layer][pg, :, off].cpu()
            assert torch.equal(got_c, wc.view(torch.uint8)), \
                f'{tag} layer {layer} {nm}: {int((got_c != wc.view(torch.uint8)).sum())} codes differ from the oracle'
            assert torch.equal(got_s, ws), f'{tag} layer {layer} {nm}: scales differ from the oracle'


def _gather(sess, row, n):
    """Row's dequantized K / V of the last layer [H, n, 64]."""
    table = sess.page_table.cpu()
    pgs = table[row, :-(-n // PAGE)].long().cuda()
    out = []
    for pool, sc in ((sess.k_pool, sess.k_scale), (sess.v_pool, sess.v_scale)):
        c = pool[-1][pgs].permute(1, 0, 2, 3).reshape(pool.shape[2], -1, 64)[:, :n]
        s = sc[-1][pgs].permute(1, 0, 2).reshape(sc.shape[2], -1)[:, :n]
        out.append(dequant(c, s))
    return out


def _check_attn(sess, cfg, q32, a16, rows_n, tag):
    """a16 rows against the float64 attention on code x scale: rows_n [(index into q32 / a16, table row, n)]."""
    Hn = cfg['num_heads']
    for i, row, n in rows_n:
        k, v = _gather(sess, row, n)
        ref, tol = fp8_attn64(q32[i:i + 1].half().view(1, Hn, 64), k.unsqueeze(0), v.unsqueeze(0))
        check(a16[i:i + 1], ref, tol, f'{tag} row {row} n={n}')


def _check_prefix(sess, slot, P, tag):
    """The slot's prefix pages (positions [0, P) of its two rows) hold the quantization of the fp16 staging cache."""
    table = sess.page_table.cpu()
    for half in range(2):
        row = half * sess.slots + slot
        for nm, stage, pool, sc in (('k', sess._stage[0], sess.k_pool, sess.k_scale),
                                    ('v', sess._stage[1], sess.v_pool, sess.v_scale)):
            wc, ws = quant_e4m3(stage[:, half, :, :P].float().cpu())
            pgs = table[row, torch.arange(P) // PAGE].long().cuda()
            offs = (torch.arange(P) % PAGE).cuda()
            got_c = pool[:, pgs, :, offs].view(torch.uint8).permute(1, 2, 0, 3).cpu()   # [P, L, H, 64] -> [L, H, P, 64]
            got_s = sc[:, pgs, :, offs].permute(1, 2, 0).cpu()
            assert torch.equal(got_c, wc.view(torch.uint8)), f'{tag}: slot {slot} prefix {nm} codes'
            assert torch.equal(got_s, ws), f'{tag}: slot {slot} prefix {nm} scales'


# (id, model, positional embedding, cross attention)
STEP_CASES = [
    ('mini-sin-nocross', 'lm_mini', 'sin', False),
    ('mini-rope-nocross', 'lm_mini', 'rope', False),
    ('mini-sin-cross', 'lm_mini', 'sin', True),
    ('mini-rope-cross', 'lm_mini', 'rope', True),
    ('melody-sin_rope', 'lm_mini_melody', 'sin_rope', False),
]
PREFIXES = (9, 63, 64, 65)


@pytest.mark.parametrize('case', STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_fp8_slot_step_and_admission(case):
    """Slots admitted at steps 0, 1 and 2 (with the melody model each with its own prefix, and its prefix pages checked
    against the staging cache at admission) sit at cache positions 63, 64 and 65 side by side at step 65; a fourth slot is
    admitted with 36 prefilled prompt columns (two passes) and its last pass is checked.  At each checkpoint step: codes and
    scales bit for bit, nothing else written, and the attention output within the bound (without cross attention)."""
    tag, name, pe, cross = case
    melody = name == 'lm_mini_melody'
    cfg, m, w = _probe_fp8(name, pe, cross, prefix=melody)
    d, Hn, slots, gen_len = cfg['dim'], cfg['num_heads'], 4, 140
    max_prefix = max(PREFIXES) if melody else 0
    kv_pages = slots * PagePool.need(max_prefix + gen_len + 8) + 6
    sess = SlotSession(m, slots, gen_len, max_text=16 if cross else 1, use_sampling=False, kv_pages=kv_pages,
                       max_prefix=max_prefix, kv_dtype='fp8')
    assert sess.k_pool.dtype == torch.float8_e4m3fn and sess.k_scale.shape == (cfg['num_layers'], kv_pages, Hn, PAGE)
    b = m._bufs
    g = torch.Generator().manual_seed(3)
    Pfx = {}

    def admit(slot, prompt_cols=0):
        cr = torch.randn(2, 5 + slot, d, generator=g) * 0.5 if cross else None
        P = PREFIXES[slot] if melody else 0
        prefix = torch.randn(2, P, d, generator=g) * 0.5 if melody else None
        prompt = None
        if prompt_cols:
            prompt = torch.randint(0, cfg['card'], (1, cfg['n_q'], prompt_cols + 4), generator=g)
        sess.admit(slot, Request(gen_len, cr, prompt, seed=slot, prefix=prefix, prefill_cols=prompt_cols))
        Pfx[slot] = P
        torch.cuda.synchronize()
        if P:
            _check_prefix(sess, slot, P, tag)

    def step_checked(label):
        st = sess.status()
        active = [s for s in range(slots) if st[s][1] == 1]
        rows_pos = [(r, Pfx[r % slots] + st[r % slots][0]) for r in range(2 * slots) if r % slots in active]
        locs = _locs(sess, rows_pos)
        keep = set()
        for r, p in rows_pos:   # the positions the step reads: [0, p) of each active row
            table = sess.page_table.cpu()
            keep.update((int(table[r, i // PAGE]), i % PAGE) for i in range(p))
        _poison(sess, keep)
        before = _snapshot(sess)
        sess.steps(1)
        torch.cuda.synchronize()
        _check_written(sess, before, locs, f'{tag} {label}')
        idx = torch.tensor([r for r, _ in rows_pos]).cuda()
        _check_codes(sess, cfg, w, b['h16'][idx], b['q32'][idx], locs, f'{tag} {label}')
        if not cross:
            _check_attn(sess, cfg, b['q32'][idx], b['a16'][idx], [(i, r, p + 1) for i, (r, p) in enumerate(rows_pos)],
                        f'{tag} {label} lm_attn2_slot_paged_fp8_kernel')
        return st

    step = 0
    for cp in (0, 1, 2, 63, 65):
        while step < cp:
            sess.steps(1)
            step += 1
        if step < 3:
            admit(step)
        step_checked(f'step {step}')
        step += 1
    st = sess.status()
    if not melody:
        assert [st[s][0] for s in range(3)] == [66, 65, 64]
    # a prefilled admission: 36 columns run as 32 + 4 positions; the last pass's q32 / h16 / a16 rows are (token, row) pairs
    # (8 of them: the session's padded rows from 8 on are zeroed after the passes)
    F = 36
    admit(3, prompt_cols=F)
    tc, p0 = F - 32, Pfx[3] + 32
    rows_pos = [(j * slots + 3, p0 + t) for t in range(tc) for j in range(2)]
    locs = _locs(sess, rows_pos)
    n = 2 * tc
    _check_codes(sess, cfg, w, b['h16'][:n], b['q32'][:n], locs, f'{tag} prefill pass')
    if not cross:
        _check_attn(sess, cfg, b['q32'][:n], b['a16'][:n], [(i, r, p + 1) for i, (r, p) in enumerate(rows_pos)],
                    f'{tag} prefill pass lm_attn2_pf_paged_fp8_kernel')
    assert sess.status()[3] == (F, 1)
    step_checked('after the prefilled admission')


@pytest.mark.parametrize('case', STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_fp8_prefill_pass(case, monkeypatch):
    """A 32-slot session (64 rows: the activation buffers hold a whole 32-position pass of one slot's two rows, none of it
    padding) admits slot 5 with 32 prefilled prompt columns, one pass, into a pool poisoned everywhere.  The admission
    writes exactly positions [0, P + 32) of the slot's two rows; every position of the pass has its codes and scales bit
    for bit, and every one of its 64 queries its attention output within the bound (without cross attention); with the
    melody model the prefix pages hold the staging cache's quantization."""
    monkeypatch.delenv('ACB_LM_PREFILL_PER', raising=False)
    tag, name, pe, cross = case
    melody = name == 'lm_mini_melody'
    cfg, m, w = _probe_fp8(name, pe, cross, prefix=melody)
    d, slots, gen_len, slot, F = cfg['dim'], 32, 80, 5, 32
    P = max(PREFIXES) if melody else 0
    sess = SlotSession(m, slots, gen_len, max_text=16 if cross else 1, use_sampling=False,
                       kv_pages=2 * PagePool.need(P + gen_len + 8) + 6, max_prefix=P, kv_dtype='fp8')
    g = torch.Generator().manual_seed(9)
    cr = torch.randn(2, 7, d, generator=g) * 0.5 if cross else None
    prefix = torch.randn(2, P, d, generator=g) * 0.5 if melody else None
    prompt = torch.randint(0, cfg['card'], (1, cfg['n_q'], F + 4), generator=g)
    _poison(sess, set())
    before = _snapshot(sess)
    sess.admit(slot, Request(gen_len, cr, prompt, seed=1, prefix=prefix, prefill_cols=F))
    torch.cuda.synchronize()
    every = _locs(sess, [(j * slots + slot, p) for j in range(2) for p in range(P + F)])
    _check_written(sess, before, every, f'{tag} admission')
    if P:
        _check_prefix(sess, slot, P, tag)
    rows_pos = [(j * slots + slot, P + t) for t in range(F) for j in range(2)]   # pass row r = t * 2 + j
    b = m._bufs
    _check_codes(sess, cfg, w, b['h16'][:2 * F], b['q32'][:2 * F], _locs(sess, rows_pos), f'{tag} prefill pass')
    if not cross:
        _check_attn(sess, cfg, b['q32'][:2 * F], b['a16'][:2 * F], [(i, r, p + 1) for i, (r, p) in enumerate(rows_pos)],
                    f'{tag} prefill pass lm_attn2_pf_paged_fp8_kernel')
    assert sess.status()[slot] == (F, 1)


# ----------------------------------------------------------------------------- end to end: mixed equals alone

def _run_fp8(mg, items, budget, prefill=True, **kw):
    gen = mg.continuous(slots=4, return_tokens=True, prefill_prompts=prefill, kv_cache_gb=budget, kv_cache_dtype='fp8',
                        **kw)
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


def _fp8_budget(mg, requests):
    from audiocraft_b200.batching import prefix_bound
    S = int(mg.max_duration * mg.frame_rate) + max(mg.lm.pattern_provider.delays) + 1
    return requests * PagePool.need(prefix_bound(mg.lm, 64) + S) * kv_page_bytes(mg.lm, 'fp8') / 1e9


def _mixed_equals_alone(mg, reqs, prefill=True):
    budget = _fp8_budget(mg, 2.5)
    items = list(enumerate(reqs))
    mixed, gen = _run_fp8(mg, items, budget, prefill)
    for i, (desc, dur, melody, prompt) in items:
        alone, _ = _run_fp8(mg, [(i, reqs[i])], budget, prefill)
        assert mixed[i][1].shape == (1, mg.lm.n_q, int(dur * mg.frame_rate))
        assert torch.equal(mixed[i][1], alone[i][1]), f'request {i} ({dur} s): fp8 tokens differ from the request alone'
        assert bool(torch.isfinite(mixed[i][0]).all())
    print(f'{mg.name}: {len(reqs)} requests equal alone in an fp8 session ({gen.session.pages.n_pages} pages, peak '
          f'{gen.session.pages.peak})')
    return mixed


def test_fp8_musicgen_requests_equal_alone(monkeypatch):
    from audiocraft_b200.musicgen import MusicGen
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    mg = _small(MusicGen.get_pretrained('synthetic/small'))
    reqs = _text_requests(mg)
    got = _mixed_equals_alone(mg, reqs)   # text, continuations and requests longer than max_duration, prompts prefilled
    short = [r for r in reqs if r[1] <= mg.max_duration]
    _mixed_equals_alone(mg, short, prefill=False)   # continuations consumed one column per step
    items = [(i, r) for i, r in enumerate(reqs) if r[1] <= mg.max_duration]
    streamed, _ = _run_fp8(mg, items, _fp8_budget(mg, 2.5), chunk_duration=0.2)
    for i, _ in items:
        assert torch.equal(streamed[i][1], got[i][1]), f'request {i}: streamed fp8 tokens differ'
        torch.testing.assert_close(streamed[i][0], got[i][0], rtol=0, atol=1e-5)


def test_fp8_melody_requests_equal_alone(monkeypatch):
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    _, _, _, mg = M._golden_musicgen()
    _mixed_equals_alone(_small(mg), _melody_requests(1))


def test_fp8_stereo_melody_requests_equal_alone(monkeypatch):
    monkeypatch.delenv('ACB_LM_PREFILL', raising=False)
    _mixed_equals_alone(_small(M._stereo_melody_musicgen()), _melody_requests(2))


def test_fp8_full_size_medium():
    """Synthetic MusicGen-medium at 64 slots with the fp8 pages of a 28 GB budget serves a mix of 96 requests to completion:
    each returns finite audio of its requested length."""
    from audiocraft_b200.loaders import load_musicgen
    mg = load_musicgen('synthetic/medium')
    gen = mg.continuous(slots=64, kv_cache_gb=28.0, kv_cache_dtype='fp8', return_tokens=True)
    assert gen.session.pages.n_pages == math.floor(28e9 / kv_page_bytes(mg.lm, 'fp8'))
    durs = {}
    for i in range(96):
        dur = [10.0, 2.0, 5.0, 8.0, 0.74][i % 5]
        durs[gen.submit(f'request {i}: a piece of music number {i}', duration=dur)] = dur
    got = {rid: (wav, tok) for rid, wav, tok in gen.run()}
    assert sorted(got) == sorted(durs)
    hop = mg.sample_rate // mg.frame_rate
    for rid, (wav, tok) in got.items():
        frames = int(durs[rid] * mg.frame_rate)
        assert tok.shape == (1, mg.lm.n_q, frames), (rid, tok.shape)
        assert wav.shape == (1, mg.audio_channels, frames * hop), (rid, wav.shape)
        assert bool(torch.isfinite(wav).all()), f'request {rid}: audio not finite'
    print(f'medium fp8, 64 slots: 96 requests with {gen.session.pages.n_pages} pages, peak {gen.session.pages.peak}, '
          f'occupancy {gen.occupancy:.2f}')
