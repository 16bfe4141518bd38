"""T5 text encoder on the device (csrc/t5.cu) against transformers' fp32 T5EncoderModel, and its share of MusicGen.generate.

    python profiles/perf_t5.py [--out DIR]

1. T5Conditioner.forward on seeded t5-base weights (output_proj to 1536, MusicGen-medium's width) for B = 1, 8, 32
   descriptions of T = 16, 64, 256 tokens, as LMModel calls it: 2B rows [cond; null], of which the B null rows are zero-filled
   without running the encoder.  CUDA events around `iters` calls after a warm-up.
2. The same rows through transformers' T5EncoderModel in fp32 (eager, on the same GPU; all 2B rows, as the reference's
   conditioner runs them) plus an fp32 output_proj and the mask, when transformers is importable.
3. MusicGen.generate(8 descriptions) on synthetic MusicGen-medium, 30 s, greedy, with the device T5 against the seeded
   precomputed-states encoder, so T5's share of the call is stated.
Prints the card name and power limit with the numbers; with --out, also writes them as JSON there.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200 import synth  # noqa: E402

SPIECE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 't5_spiece.model')
DESCS = ['calm piano melody with soft strings', 'heavy techno beat with deep bass', 'jazz saxophone solo at night',
         'orchestral epic cinematic choir', 'lofi hip hop chill beat with rain', 'upbeat electronic synth pad',
         'slow sad violin and cello', 'fast drums and guitar solo']


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name()


def event_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def inputs_for(B, T, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, 32000, (2 * B, T), generator=g)
    mask = torch.zeros(2 * B, T, dtype=torch.long)
    mask[:B] = 1
    ids[B:] = 0
    ids[B:, 0] = 1
    return {'input_ids': ids, 'attention_mask': mask}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    os.environ.setdefault('HF_HUB_OFFLINE', '1')
    torch.set_grad_enabled(False)
    from audiocraft_b200.conditioners import T5Conditioner
    info = gpu_info()
    print('GPU:', info)
    res = {'gpu': info, 'encode': [], 'generate': {}}
    cfg = synth.t5_config('t5-base')
    with tempfile.TemporaryDirectory() as tmp:
        sd = synth.synth_t5_state_dict(cfg, seed=1)
        synth.write_t5_dir(tmp, cfg, sd, SPIECE)
        cond = T5Conditioner(tmp, 1536, device='cuda').to('cuda')
        hf = None
        try:
            from transformers import T5Config, T5EncoderModel
            hf = T5EncoderModel(T5Config(**{k: v for k, v in cfg.items() if k != 'model_type'})).eval()
            hf.load_state_dict(sd, strict=False)
            hf = hf.cuda()
            proj = cond.output_proj
        except ImportError:
            print('transformers not importable: no comparator')
        print(f"{'B':>3} {'T':>4} {'rows':>5}  {'device ms':>10} {'transformers ms':>16}")
        for B in (1, 8, 32):
            for T in (16, 64, 256):
                inp = inputs_for(B, T)
                dev = event_ms(lambda: cond(inp), args.iters)
                ref = None
                if hf is not None:
                    ids, mask = inp['input_ids'].cuda(), inp['attention_mask'].cuda()

                    def run_hf():
                        h = hf(input_ids=ids, attention_mask=mask).last_hidden_state
                        return proj(h) * mask.unsqueeze(-1)
                    ref = event_ms(run_hf, args.iters)
                res['encode'].append(dict(B=B, T=T, rows=2 * B, device_ms=dev, transformers_fp32_ms=ref))
                print(f"{B:>3} {T:>4} {2 * B:>5}  {dev:>10.3f} {ref if ref is None else round(ref, 3):>16}")
        del hf

        from audiocraft_b200.musicgen import MusicGen
        for arm, enc in (('device_t5', tmp), ('precomputed', None)):
            model = MusicGen.get_pretrained('synthetic/medium', text_encoder=enc)
            model.set_generation_params(use_sampling=False, duration=30)
            model.generate(DESCS[:2])   # warm-up: graph capture, tokenizer, first launches
            times = []
            for _ in range(2):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.generate(DESCS)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            res['generate'][arm] = times
            print(f"MusicGen.generate synthetic medium 30 s B=8 ({arm}): {min(times):.3f} s (runs {', '.join(f'{t:.3f}' for t in times)})")
            del model
            torch.cuda.empty_cache()
        share = min(res['generate']['device_t5']) - min(res['generate']['precomputed'])
        print(f"T5 share of generate: {share * 1e3:.1f} ms of {min(res['generate']['device_t5']):.3f} s")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'perf_t5.json'), 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
