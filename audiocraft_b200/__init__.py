"""audiocraft_b200 -- H100-native (sm_90a) implementation of AudioCraft's two inference hot paths behind the
reference's Python API: EnCodec (SEANet + RVQ) encode/decode and MusicGen LM autoregressive decode."""
__version__ = '0.1.0'
