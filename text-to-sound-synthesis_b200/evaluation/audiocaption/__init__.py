"""Drop-ins for the reference Codebook/AudiocaptionLoss: the ACT captioning transformer (models/TransModel.py, models/AudioTransformer.py) and
its greedy and beam decoders (tools/utils.py greedy_decode, tools/beam.py beam_decode), run on the sm_90a kernels by caption_engine."""
from .models import ACT, AudioTransformer_80, PositionalEncoding
from .decode import BeamSearchNode, beam_decode, beam_search, greedy_decode

__all__ = ["ACT", "AudioTransformer_80", "PositionalEncoding", "BeamSearchNode", "beam_decode", "beam_search", "greedy_decode"]
