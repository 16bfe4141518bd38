"""Generate the stereo MusicGen fixtures by running the REAL reference modules on the CPU in fp32 (found through
oracle/ref_import.py: $AUDIOCRAFT_REFERENCE or baseline/_ref).

    python tests/golden/make_golden_stereo.py [mini|full]      (both without an argument)

* tests/golden/lm_mini_stereo.pt (`mini`): the reference's LMModel at n_q = 8 with the paired delays [0,0,1,1,2,2,3,3] of
  the stereo checkpoints (lm_mini_stereo: d = 256, card 2048, so the heads are n_q * card = 16384 wide) --
  greedy tokens, a greedy continuation of a 5-frame prompt, the CFG-mixed teacher-forced logits of one causal forward along
  the greedy sequence, and compute_predictions with and without keep_only_valid_steps; and the reference's
  InterleaveStereoCompressionModel (per_timestep false) over a seeded encodec_32k codec: codes and decoded waveform.
* tests/golden/musicgen_stereo_medium_full.pt (`full`): full-depth MusicGen-stereo-medium, one causal forward over a
  1500-frame delay-pattern sequence with rows [cond; null], top-32 CFG-mixed logits at the kept steps (the format of
  musicgen_medium_full.pt, make_golden.py golden_lm_fullsize).

Weights, conditions, codes and audio are regenerated from the seeds stored beside the outputs (audiocraft_b200/synth.py,
tests/helpers.py); only outputs are stored, the float logits at a seeded sample of card indices to keep the fixture small.
"""
import os
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import ref_import as R  # noqa: E402
from oracle.ref_models import build_ref_encodec, build_ref_lm, text_table  # noqa: E402
from tests import helpers as H  # noqa: E402
from audiocraft_b200 import synth  # noqa: E402

warnings.filterwarnings('ignore')
torch.set_grad_enabled(False)

NAME = 'lm_mini_stereo'
WSEED, CSEED, SSEED, KSEED, IDX_SEED, N_IDX = 3, 1, 5, 8, 11, 64
B, T_TEXT, T, T_PRED, PROMPT = 2, 5, 12, 20, 5
PRED_TOPN = 16
CODEC, CODEC_WSEED, CODEC_XSEED, CODEC_LEN, WAV_STRIDE = 'encodec_32k', 7, 9, 16000, 37
FULL_STEPS = [0, 1, 374, 749, 1124, 1499, 1502]


def golden_mini():
    cfg = synth.lm_config(NAME)
    sd = synth.synth_lm_state_dict(cfg, seed=WSEED)
    hid, mask, cross = H.lm_condition(cfg, sd, B, T_TEXT, CSEED)
    m, CA = build_ref_lm(cfg, sd, text_table(hid, mask, cfg['cond_dim']))
    conds = [CA(text={'description': f'd{i}'}) for i in range(B)]
    idx = torch.randperm(cfg['card'], generator=torch.Generator().manual_seed(IDX_SEED))[:N_IDX].sort().values
    out = dict(name=NAME, batch=B, t_text=T_TEXT, T=T, wseed=WSEED, cseed=CSEED, logits_idx=idx)

    greedy = m.generate(None, conds, max_gen_len=T, use_sampling=False)                     # [B, 8, T]
    out['greedy'] = greedy
    out['continuation'] = m.generate(greedy[..., :PROMPT].clone(), conds, max_gen_len=T, use_sampling=False)
    out['prompt_len'] = PROMPT
    # CFG-mixed logits of one causal forward over the greedy delay-pattern sequence: what the decode step computes at
    # each position when it is teacher-forced along that sequence
    pat = m.pattern_provider.get_pattern(T)
    seq = pat.build_pattern_sequence(greedy, m.special_token_id)[0]                          # [B, 8, T + 4]
    ct = {'description': (cross, torch.ones(cross.shape[:2], dtype=torch.long))}
    lg = m(torch.cat([seq, seq], 0)[..., :-1], conditions=[], condition_tensors=ct)          # [2B, 8, S-1, card]
    c, u = lg.split(B, dim=0)
    mixed = (u + (c - u) * cfg['cfg_coef']).permute(2, 0, 1, 3).contiguous()                 # [S-1, B, 8, card]
    top2 = mixed.topk(2, dim=-1).values
    out.update(sequence=seq, logits=mixed[..., idx].clone(), logits_argmax=mixed.argmax(-1).to(torch.int16),
               logits_margin=(top2[..., 0] - top2[..., 1]).clone())

    codes = torch.randint(0, cfg['card'], (B, cfg['n_q'], T_PRED), generator=torch.Generator().manual_seed(KSEED))
    pred = dict(T=T_PRED, kseed=KSEED, topn=PRED_TOPN)
    for valid in (True, False):
        o = m.compute_predictions(codes, conds, keep_only_valid_steps=valid)
        key = 'valid' if valid else 'all'
        pred[f'mask_{key}'] = o.mask[0].clone()
        pred[f'nan_{key}'] = torch.isnan(o.logits[..., 0]).clone()
        v, i = torch.nan_to_num(o.logits, nan=-1e30).topk(PRED_TOPN, dim=-1)
        pred[f'top_v_{key}'], pred[f'top_i_{key}'] = v.clone(), i.to(torch.int16)
        pred[f'logits_{key}'] = o.logits[..., idx].clone()
    out['predictions'] = pred

    ccfg = synth.ENCODEC_CONFIGS[CODEC]
    enc = R.mod('models.encodec')
    wrapped = enc.InterleaveStereoCompressionModel(build_ref_encodec(ccfg, synth.synth_encodec_state_dict(ccfg, seed=CODEC_WSEED)),
                                                   per_timestep=False)
    x = H.audio_input(dict(ccfg, channels=2), B, CODEC_LEN, CODEC_XSEED)
    ccodes, scale = wrapped.encode(x)
    assert scale is None
    wav = wrapped.decode(ccodes, None)
    out['codec'] = dict(name=CODEC, wseed=CODEC_WSEED, xseed=CODEC_XSEED, length=CODEC_LEN, x_head=x[..., :64].clone(),
                        codes=ccodes, wav_len=wav.shape[-1], wav_stride=WAV_STRIDE, wav_strided=wav[..., ::WAV_STRIDE].clone(),
                        props=(wrapped.num_codebooks, wrapped.frame_rate, wrapped.channels, wrapped.cardinality,
                               wrapped.total_codebooks))
    torch.save(out, os.path.join(H.GOLDEN_DIR, f'{NAME}.pt'))
    print(NAME, 'greedy', tuple(greedy.shape), 'logits', tuple(out['logits'].shape), 'codec codes', tuple(ccodes.shape),
          'wav', tuple(wav.shape))


def golden_full(name='musicgen_stereo_medium', batch=4, t_text=16, T_full=1500, wseed=0, cseed=3, sseed=17, topn=32):
    t0 = time.time()
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=wseed)
    _, _, cross = H.lm_condition(cfg, sd, batch, t_text, cseed)
    m, _ = build_ref_lm(cfg, sd, {'__null__': (torch.zeros(t_text, cfg['cond_dim']), torch.zeros(t_text, dtype=torch.long))})
    del sd
    seq = H.fullsize_sequence(cfg, batch, T_full, sseed)                  # [B, 8, T + 4]
    S = seq.shape[-1]
    ct = {'description': (cross, torch.ones(cross.shape[:2], dtype=torch.long))}
    logits = m(torch.cat([seq, seq], 0)[..., :S - 1], conditions=[], condition_tensors=ct)   # [2B, 8, S-1, card]
    c, u = logits.split(batch, dim=0)
    mixed = (u + (c - u) * cfg['cfg_coef'])[:, :, FULL_STEPS, :].permute(2, 0, 1, 3).contiguous()   # [n, B, 8, card]
    tv, ti = mixed.topk(topn, dim=-1)
    out = dict(name=name, batch=batch, t_text=t_text, T=T_full, wseed=wseed, cseed=cseed, sseed=sseed, steps=FULL_STEPS,
               logits_top_v=tv, logits_top_i=ti.to(torch.int16), seq_head=seq[..., :16].clone())
    torch.save(out, os.path.join(H.GOLDEN_DIR, f'{name}_full.pt'))
    print(name, 'fullsize logits', tuple(tv.shape), f'{time.time() - t0:.0f} s')


if __name__ == '__main__':
    what = sys.argv[1] if len(sys.argv) > 1 else 'both'
    if what in ('mini', 'both'):
        golden_mini()
    if what in ('full', 'both'):
        golden_full()
