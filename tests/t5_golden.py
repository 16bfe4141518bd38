"""What tests/golden/t5_conditioner.pt was made from (tests/golden/make_golden_t5.py), shared with the tests that read it.

Weights are regenerated from seeds (audiocraft_b200.synth.synth_t5_state_dict); the tokenizer is the small SentencePiece model
tests/golden/t5_spiece.model, trained offline by the generator (T5's special ids: pad 0, eos 1, unk 2)."""
import os

import torch

from audiocraft_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 't5_conditioner.pt')
SPIECE = os.path.join(HERE, 'golden', 't5_spiece.model')
SAMPLES = 384   # values stored per row and tensor (seeded positions)

WORDS = ("calm piano melody with soft strings ambient drone techno beat heavy bass drums guitar solo jazz saxophone "
         "orchestral epic cinematic lofi hip hop chill rain thunder birds chirping dog barking car engine crowd cheering "
         "upbeat happy sad slow fast electronic synth pad violin cello flute choir vocals whistle wind ocean waves footsteps")

LONG = ' '.join(WORDS.split()[i % 17] + ('s' if i % 3 == 0 else '') for i in range(90)) + ' Quirky XYLOPHONE 1977!'

# name -> (T5 architecture, weight seed, wi scale, output_proj out_dim, proj seed, descriptions, hand-made id rows)
CASES = {
    # MusicGen (text2music.yaml): prompts of several lengths, None and "" entries, one prompt past 128 tokens
    'base': ('t5-base', 11, 1.0, 1536, 21,
             ['calm piano melody with soft strings', None, 'heavy techno beat', '', LONG, 'jazz saxophone solo at night'], 3),
    # AudioGen (text2sound.yaml)
    'large': ('t5-large', 12, 1.0, 1536, 22, ['dog barking in the rain', 'car engine', None], 0),
    # wi scaled so that ReLU activations pass fp16's 65504 (the generator asserts it)
    'hot': ('t5-base', 13, 3.0e4, 1536, 23, ['orchestral epic cinematic choir', 'birds chirping', ''], 0),
}


def proj_weights(d_model: int, out_dim: int, seed: int):
    """The conditioner's output_proj (nn.Linear(d_model, out_dim)) weight and bias."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn((out_dim, d_model), generator=g) * d_model ** -0.5, 0.05 * torch.randn(out_dim, generator=g)


def state_dict(case: str):
    arch, seed, wi_scale = CASES[case][:3]
    cfg = synth.t5_config(arch)
    return cfg, synth.synth_t5_state_dict(cfg, seed, wi_scale)


def hand_ids(n_rows: int, T: int = 40, seed: int = 31):
    """Token ids spread over the whole 32128-row embedding with ragged masks (row r keeps T - 7 r tokens)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 32128, (n_rows, T), generator=g)
    mask = (torch.arange(T)[None, :] < (T - 7 * torch.arange(n_rows))[:, None]).long()
    return ids, mask


def sample_index(rows: int, inner: int, seed: int):
    """[rows][SAMPLES] seeded flat positions into each row's [T * dim] values."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, inner, (rows, SAMPLES), generator=g)
