"""Generate tests/golden/lm_predictions.pt: the REAL reference's LMModel.compute_predictions / forward on CPU in fp32
(oracle/ref_models.py), and its Pattern.revert_pattern_logits index tables.

    python tests/golden/make_golden_predictions.py

Weights, codes and text conditions are regenerated from the seeds stored next to the outputs (tests/helpers.py,
audiocraft_b200/synth.py); only outputs are stored.  MusicGen-small keeps the top-32 logits per position to stay small.
"""
import os
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import ref_import as R  # noqa: E402
from oracle.ref_models import build_ref_lm, text_table  # noqa: E402
from tests import helpers as H  # noqa: E402
from audiocraft_b200 import synth  # noqa: E402

warnings.filterwarnings('ignore')
torch.set_grad_enabled(False)

# (name, batch, t_text, T, wseed, cseed, codes seed, top-n or None)
CASES = [('lm_tiny', 2, 5, 23, 3, 4, 5, None),
         ('lm_mini', 3, 7, 37, 6, 7, 8, None),
         ('musicgen_small', 2, 9, 40, 9, 10, 11, 32)]
TABLES = [(4, 11, [0, 1, 2, 3]), (8, 9, [0, 0, 1, 1, 2, 2, 3, 3]), (3, 6, [0, 0, 2])]


def codes_for(cfg, batch, T, seed):
    return torch.randint(0, cfg['card'], (batch, cfg['n_q'], T), generator=torch.Generator().manual_seed(seed))


def main():
    out = {'cases': {}, 'tables': {}}
    for name, B, t_text, T, wseed, cseed, kseed, topn in CASES:
        cfg = synth.lm_config(name)
        sd = synth.synth_lm_state_dict(cfg, seed=wseed)
        hid, mask, _ = H.lm_condition(cfg, sd, B, t_text, cseed)
        m, CA = build_ref_lm(cfg, sd, text_table(hid, mask, cfg['cond_dim']))
        conds = [CA(text={'description': f'd{i}'}) for i in range(B)]
        codes = codes_for(cfg, B, T, kseed)
        case = dict(batch=B, t_text=t_text, T=T, wseed=wseed, cseed=cseed, kseed=kseed, topn=topn)
        for valid in (True, False):
            o = m.compute_predictions(codes, conds, keep_only_valid_steps=valid)
            key = 'valid' if valid else 'all'
            case[f'mask_{key}'] = o.mask[0].clone()
            lg = o.logits
            case[f'nan_{key}'] = torch.isnan(lg[..., 0]).clone()
            if topn is None:
                case[f'logits_{key}'] = lg.clone()
            else:
                v, i = torch.nan_to_num(lg, nan=-1e30).topk(topn, dim=-1)
                case[f'top_v_{key}'], case[f'top_i_{key}'] = v.clone(), i.to(torch.int16)
        out['cases'][name] = case
        print(name, 'logits', tuple(o.logits.shape))
    pat = R.mod('modules.codebooks_patterns')
    for K, T, delays in TABLES:
        p = pat.DelayedPatternProvider(K, delays=delays).get_pattern(T)
        tabs = {}
        for valid in (True, False):
            S = p.build_pattern_sequence(torch.zeros(1, K, T, dtype=torch.long), 0, keep_only_valid_steps=valid)[0].shape[-1]
            for s in sorted({S, max(1, S - 2)}):
                idx, msk = p._build_reverted_sequence_scatter_indexes(s, K, valid, is_model_output=True)
                tabs[(valid, s)] = (idx.clone(), msk.clone())
        out['tables'][(K, T, tuple(delays))] = tabs
    torch.save(out, os.path.join(H.GOLDEN_DIR, 'lm_predictions.pt'))
    print('tables', len(out['tables']))


if __name__ == '__main__':
    main()
