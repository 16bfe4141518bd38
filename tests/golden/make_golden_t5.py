"""Generate tests/golden/t5_conditioner.pt (and the tokenizer model tests/golden/t5_spiece.model): the REAL reference's
T5Conditioner (audiocraft/modules/conditioners.py:422-515) on CPU in fp32, with its transformers T5Tokenizer and
T5EncoderModel.

    python tests/golden/make_golden_t5.py

There are no pretrained T5 weights offline, so `from_pretrained` is patched to build locally: the tokenizer from a small
SentencePiece model trained here, the encoder from transformers' T5Config of the named architecture with seeded weights
(audiocraft_b200.synth.synth_t5_state_dict).  Cases: tests/t5_golden.py.  For each, the conditioner tokenizes
[descriptions; None per description] (the [cond; null] rows LMModel builds) and the stored outputs are the ids, the masks,
and SAMPLES seeded values per row of T5's last_hidden_state and of the conditioner's output.
"""
import os
import random
import shutil
import sys
import tempfile
import warnings
from unittest import mock

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import ref_import as R  # noqa: E402
from tests import t5_golden as G  # noqa: E402

warnings.filterwarnings('ignore')
torch.set_grad_enabled(False)


def train_spiece(path: str):
    import sentencepiece as spm
    rnd = random.Random(0)
    words = G.WORDS.split()
    lines = [' '.join(rnd.choice(words) for _ in range(rnd.randint(3, 12))) for _ in range(3000)]
    with tempfile.TemporaryDirectory() as tmp:
        prefix = os.path.join(tmp, 'sp')
        spm.SentencePieceTrainer.train(sentence_iterator=iter(lines), model_prefix=prefix, vocab_size=200, model_type='unigram',
                                       pad_id=0, eos_id=1, unk_id=2, bos_id=-1, character_coverage=1.0,
                                       hard_vocab_limit=False, minloglevel=2)
        shutil.copyfile(prefix + '.model', path)


def main():
    if not os.path.exists(G.SPIECE):
        train_spiece(G.SPIECE)
    from transformers import T5Config, T5EncoderModel, T5Tokenizer
    cond_mod = R.mod('modules.conditioners')
    tok_dir = tempfile.mkdtemp()
    shutil.copyfile(G.SPIECE, os.path.join(tok_dir, 'spiece.model'))
    tokenizer = T5Tokenizer.from_pretrained(tok_dir, local_files_only=True)
    out = {'cases': {}}
    for name, (arch, seed, wi_scale, out_dim, pseed, descs, n_hand) in G.CASES.items():
        cfg, sd = G.state_dict(name)
        enc = T5EncoderModel(T5Config(**{k: v for k, v in cfg.items() if k != 'model_type'})).eval()
        missing, unexpected = enc.load_state_dict(sd, strict=False)
        assert not unexpected and all('embed_tokens' in k for k in missing), (missing, unexpected)
        with mock.patch.object(T5Tokenizer, 'from_pretrained', lambda *a, **k: tokenizer), \
                mock.patch.object(T5EncoderModel, 'from_pretrained', lambda *a, **k: enc):
            cond = cond_mod.T5Conditioner(arch, out_dim, finetune=False, device='cpu')
        pw, pb = G.proj_weights(cfg['d_model'], out_dim, pseed)
        cond.output_proj.weight.copy_(pw)
        cond.output_proj.bias.copy_(pb)
        act_max = [0.0]
        hooks = [b.layer[1].DenseReluDense.act.register_forward_hook(
            lambda m, i, o: act_max.__setitem__(0, max(act_max[0], float(o.max())))) for b in enc.encoder.block]
        inputs = cond.tokenize(list(descs) + [None] * len(descs))
        emb, mask = cond(inputs)
        hid = enc(**inputs).last_hidden_state
        for h in hooks:
            h.remove()
        case = dict(arch=arch, seed=seed, wi_scale=wi_scale, out_dim=out_dim, pseed=pseed, descs=list(descs),
                    ids=inputs['input_ids'].clone(), mask=mask.clone(), act_max=act_max[0])
        rows, T = inputs['input_ids'].shape
        hi, ei = G.sample_index(rows, T * cfg['d_model'], seed + 100), G.sample_index(rows, T * out_dim, seed + 200)
        case['hid_idx'], case['hid'] = hi.to(torch.int32), hid.reshape(rows, -1).gather(1, hi).clone()
        case['emb_idx'], case['emb'] = ei.to(torch.int32), emb.reshape(rows, -1).gather(1, ei).clone()
        if n_hand:
            ids, hm = G.hand_ids(n_hand)
            he, _ = cond({'input_ids': ids, 'attention_mask': hm})
            hh = enc(input_ids=ids, attention_mask=hm).last_hidden_state
            Th = ids.shape[1]
            hi, ei = G.sample_index(n_hand, Th * cfg['d_model'], seed + 300), G.sample_index(n_hand, Th * out_dim, seed + 400)
            case['hand'] = dict(ids=ids, mask=hm, hid_idx=hi.to(torch.int32), hid=hh.reshape(n_hand, -1).gather(1, hi).clone(),
                                emb_idx=ei.to(torch.int32), emb=he.reshape(n_hand, -1).gather(1, ei).clone())
        if name == 'hot':
            assert act_max[0] > 65504, f"hot case: largest ReLU activation {act_max[0]:.0f} does not pass fp16's range"
        out['cases'][name] = case
        print(f"{name}: {arch} rows {rows} T {T} |hidden| max {hid.abs().max():.3g} relu max {act_max[0]:.3g}")
    shutil.rmtree(tok_dir)
    torch.save(out, G.GOLDEN)
    print('wrote', G.GOLDEN, os.path.getsize(G.GOLDEN), 'bytes')


if __name__ == '__main__':
    main()
