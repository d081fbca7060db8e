"""Writes tests/golden/act_ref.npz and tests/golden/act_state_dict_keys.json from the UNMODIFIED reference Codebook/AudiocaptionLoss, run on the
CPU in fp32.  gensim, h5py, librosa and dotmap are absent here, so stub modules stand in for the imports the reference's tools package makes (ACT only
calls gensim with
word_embedding.pretrained, which these configs leave off); the config is a namespace instead of a DotMap.  Weights and mels come from
oracle.act_oracle's hash recipe, so the fixture stores only the seeds.

Cases, clips 22 and 55 of seeded_mels(21, 64), 80 x 848 each:
  full:  nhid 512, 4 layers, 8 heads, V = 5000 (the released settings.yaml decoder); encoder memory, teacher-forced forward logits, greedy ids
         (max_len 30) and beam_decode ids for beam 2 and 3 with the <eos> logit biased by 2.3: at beam 2 clip 22 ends on
         <eos> after 26 words and clip 55 stops at the cap after 172; at beam 3 clip 55 ends after 20 words and clip 22 stops at the cap
         after 24;
  cap:   nhid 128, 1 layer, 2 heads, V = 5000, no bias: beam_decode for beam 2 and 3 runs into the qsize > 2000 cut-off."""
import json
import os
import sys
import types
from types import SimpleNamespace as NS

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import act_oracle as O  # noqa: E402

REF = os.path.join(os.environ.get("DIFFSOUND_REFERENCE", "/root/reference"), "Codebook", "AudiocaptionLoss")
V, SOS, EOS = 5000, 0, 9
CASES = dict(full=dict(nhid=512, nlayers=4, nhead=8, ff=2048, seed=11, eos_bias=2.3), cap=dict(nhid=128, nlayers=1, nhead=2, ff=512, seed=12, eos_bias=0.0))
MEL_SEED, MEL_CLIPS, TGT = 21, [22, 55], [[SOS, 17, 4, 250, 3999, 9, 77, 1000], [SOS, 1, 2, 3, 4, 5, 6, 4999]]


def config(c):
    return NS(encoder=NS(model="audioset", freeze=False, pretrained=False),
              decoder=NS(nhead=c["nhead"], nhid=c["nhid"], nlayers=c["nlayers"], dropout=0.2, dim_feedforward=c["ff"], activation="gelu"),
              word_embedding=NS(pretrained=False, freeze=False), path=NS())


def main():
    for absent in ("h5py", "librosa", "dotmap"):  # tools/__init__.py imports them; nothing here reads .h5 files, audio or YAML configs
        sys.modules.setdefault(absent, types.ModuleType(absent))
    sys.modules["dotmap"].DotMap = dict
    sys.modules.setdefault("gensim", types.ModuleType("gensim"))
    w2v = types.ModuleType("gensim.models.word2vec")
    w2v.Word2Vec = None
    sys.modules.setdefault("gensim.models", types.ModuleType("gensim.models"))
    sys.modules.setdefault("gensim.models.word2vec", w2v)
    sys.path.insert(0, REF)
    from models.TransModel import ACT
    from tools.beam import beam_decode
    from tools.utils import greedy_decode
    torch.set_num_threads(os.cpu_count() or 1)
    mels = O.seeded_mels(MEL_SEED, 64)[MEL_CLIPS]
    out, keys = {}, None
    for name, c in CASES.items():
        model = ACT(config(c), V).eval()
        sd = O.seeded_state_dict(model.state_dict(), c["seed"], EOS, c["eos_bias"])
        model.load_state_dict(sd)
        if keys is None:
            keys = [[k, list(v.shape)] for k, v in model.state_dict().items()]
        with torch.no_grad():
            if name == "full":
                out["full_memory"] = model.encode(mels).transpose(0, 1).numpy()
                out["full_forward"] = model(mels, torch.tensor(TGT)).transpose(0, 1).numpy()
                out["full_greedy"] = greedy_decode(model, mels, SOS, EOS, max_len=30).numpy()
            for bw in (2, 3):
                ids = beam_decode(mels, model, SOS, EOS, beam_width=bw, top_k=1).numpy()
                out[f"{name}_beam{bw}"] = ids
                print(name, bw, ids.shape, ids[:, :24].tolist(), flush=True)
    out["tgt"] = np.array(TGT)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "act_ref.npz"), **out)
    with open(os.path.join(ROOT, "tests", "golden", "act_state_dict_keys.json"), "w") as f:
        json.dump(keys, f, indent=0)


if __name__ == "__main__":
    main()
