"""The shared engine lifecycle (engine_base.PackedEngine / EngineModule) on the CPU: when packed copies are rebuilt and what a deep copy keeps."""
import copy

import pytest
import torch
from torch import nn

import _pkg

_pkg.load()
from diffsound_b200.engine_base import EngineModule, PackedEngine  # noqa: E402


class _CountingEngine(PackedEngine):
    settings = ("use_cuda_graph",)

    def __init__(self, module, scale=1.0):
        super().__init__(module, scale=scale)
        self.scale = scale
        self.use_cuda_graph = True
        self.packs = 0

    def _pack(self):
        self.packs += 1


class _Host(EngineModule):
    def __init__(self):
        super().__init__()
        self.lin = nn.Linear(4, 3)
        self.register_buffer("stat", torch.zeros(3))
        self.engine = _CountingEngine(self, scale=2.0)


def _current(m):
    """ensure_current() and the number of _pack() calls it made."""
    n = m.engine.packs
    m.engine.ensure_current()
    return m.engine.packs - n


def test_first_call_packs_and_a_second_does_not():
    m = _Host()
    assert not m.engine.packed and m.engine.generation == 0
    assert _current(m) == 1 and m.engine.packed
    assert _current(m) == 0


@pytest.mark.parametrize("change", ["inplace_parameter", "inplace_buffer", "load_state_dict", "double"])
def test_changes_repack(change):
    m = _Host()
    _current(m)
    if change == "inplace_parameter":
        with torch.no_grad():
            m.lin.weight.mul_(1.01)
    elif change == "inplace_buffer":
        m.stat.add_(1.0)
    elif change == "load_state_dict":
        m.load_state_dict({k: v + 1 for k, v in m.state_dict().items()})
    else:
        m.double()  # any _apply (.to() / .cuda() / .cpu() / .double()) marks the engines unpacked
        assert not m.engine.packed
    assert _current(m) == 1
    assert _current(m) == 0


def test_writes_through_data_need_an_explicit_repack():
    m = _Host()
    _current(m)
    m.lin.weight.data.copy_(torch.ones(3, 4))  # bypasses the version counter: not detected
    assert _current(m) == 0
    m.engine.packed = False
    assert _current(m) == 1
    m.lin.bias.data.zero_()
    m.engine.repack()
    assert m.engine.packs == 3 and _current(m) == 0


def test_generation_counts_repacks():
    m = _Host()
    for i in range(1, 4):
        m.engine.repack()
        assert m.engine.generation == i
    with torch.no_grad():
        m.lin.bias.add_(1.0)
    _current(m)
    assert m.engine.generation == 4


def test_deepcopy_gives_an_unpacked_engine_on_the_copy():
    m = _Host()
    _current(m)
    m.engine.use_cuda_graph = False
    cp = copy.deepcopy(m)
    e = cp.engine
    assert type(e) is _CountingEngine and e is not m.engine and e.m is cp
    assert not e.packed and e.packs == 0 and e.generation == 0
    assert e.options == {"scale": 2.0} and e.scale == 2.0 and e.use_cuda_graph is False
    assert torch.equal(cp.lin.weight, m.lin.weight) and cp.lin.weight.data_ptr() != m.lin.weight.data_ptr()
    assert _current(cp) == 1 and _current(m) == 0


def test_every_inference_engine_is_a_packed_engine():
    from diffsound_b200.ar_engine import AREngine
    from diffsound_b200.caption_engine import CaptionEngine
    from diffsound_b200.decoder_engine import DecoderEngine
    from diffsound_b200.encoder_engine import EncoderEngine
    from diffsound_b200.engine import DenoiserEngine
    from diffsound_b200.melception_engine import MelceptionEngine
    from diffsound_b200.text_engine import TextTowerEngine
    from diffsound_b200.vocoder_engine import VocoderEngine
    for cls in (DenoiserEngine, AREngine, CaptionEngine, MelceptionEngine, DecoderEngine, EncoderEngine, VocoderEngine, TextTowerEngine):
        assert issubclass(cls, PackedEngine), cls.__name__
