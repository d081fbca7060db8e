"""ACT audio captioning without a GPU: the oracle against the reference's fixtures, the drop-in's host beam search driven by the oracle's
log-probs, the state_dict layout, refusals, the caption tool's dry run and the new kernels' register use."""
import json
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200.evaluation.audiocaption import ACT, beam_search  # noqa: E402
from oracle import act_oracle as O  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
V, SOS, EOS = 5000, 0, 9
CASES = dict(full=dict(nhid=512, nlayers=4, nhead=8, ff=2048, seed=11, eos_bias=2.3), cap=dict(nhid=128, nlayers=1, nhead=2, ff=512, seed=12, eos_bias=0.0))


def fixture_mels():
    """The two clips of the fixtures (oracle/gen_golden_act.py)."""
    return O.seeded_mels(21, 64)[[22, 55]]


def config(c, **kw):
    return NS(encoder=NS(model="audioset", freeze=False, pretrained=False),
              decoder=NS(nhead=c["nhead"], nhid=c["nhid"], nlayers=c["nlayers"], dropout=0.2, dim_feedforward=c["ff"], activation="gelu"),
              word_embedding=NS(pretrained=kw.get("w2v", False), freeze=False), path=NS(vocabulary="words.p", word2vec="w2v.model"))


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(os.path.join(GOLD, "act_ref.npz")))


def _sd(name):
    c = CASES[name]
    return O.seeded_state_dict(ACT(config(c), V).state_dict(), c["seed"], EOS, c["eos_bias"]), c


def test_state_dict_matches_reference():
    with open(os.path.join(GOLD, "act_state_dict_keys.json")) as f:
        want = [tuple([k, tuple(s)]) for k, s in json.load(f)]
    got = [(k, tuple(v.shape)) for k, v in ACT(config(CASES["full"]), V).state_dict().items()]
    assert got == want and len(got) == 235


def test_train_mode_and_missing_gensim_refused():
    m = ACT(config(CASES["cap"]), V)
    with pytest.raises(NotImplementedError, match="inference only"):
        m.encode(torch.zeros(1, 848, 80))
    try:
        import gensim  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="gensim"):
            ACT(config(CASES["cap"], w2v=True), V)


@pytest.fixture(scope="module")
def memories():
    mels = fixture_mels()
    return {name: O.encode(_sd(name)[0], mels) for name in CASES}


def test_oracle_matches_reference(ref, memories):
    sd, c = _sd("full")
    mem = memories["full"]
    np.testing.assert_allclose(mem.numpy(), ref["full_memory"], rtol=0, atol=2e-4 * float(np.abs(ref["full_memory"]).max()))
    logits = O.decode(sd, mem, torch.from_numpy(ref["tgt"]), c["nhead"])
    np.testing.assert_allclose(logits.numpy(), ref["full_forward"], rtol=0, atol=2e-4 * float(np.abs(ref["full_forward"]).max()))
    assert np.array_equal(O.greedy_decode(sd, mem, c["nhead"], SOS, 30).numpy(), ref["full_greedy"])


@pytest.mark.parametrize("name,bw", [("full", 2), ("full", 3), ("cap", 2), ("cap", 3)])
def test_host_search_reproduces_reference(ref, memories, name, bw):
    """beam_search with every clip in one round, driven by the oracle's fp64 log-probs rounded to fp32, returns the reference's ids."""
    sd, c = _sd(name)
    mem = memories[name]
    cache = {}

    def expand(items):
        vals, idx = [], []
        for clip, node in items:
            words = tuple(node.words())
            if (clip, words) not in cache:
                lp = O.next_logprobs(sd, mem[clip], list(words), c["nhead"]).float()
                v, i = torch.topk(lp, bw)
                cache[(clip, words)] = (v.tolist(), i.tolist())
            vals.append(cache[(clip, words)][0])
            idx.append(cache[(clip, words)][1])
        return vals, idx

    seqs = beam_search(expand, 2, SOS, EOS, bw, 1)
    want = ref[f"{name}_beam{bw}"]
    got = np.full((len(seqs), max(len(s) for s in seqs)), EOS)
    for r, s in enumerate(seqs):
        got[r, :len(s)] = s
    assert got.shape == want.shape and np.array_equal(got, want)


def test_host_search_matches_oracle_search_per_clip():
    """The batched host search equals the reference algorithm (PriorityQueue, one clip at a time) on synthetic log-probs with exact ties."""
    rng = np.random.default_rng(3)
    table = {}

    def lp_of(clip, words):
        key = (clip, tuple(words))
        if key not in table:
            v = np.sort(rng.choice(np.arange(-40, -1) / 10, 6, replace=False))[::-1]  # one decimal: equal scores and logp between nodes
            table[key] = (v.astype(np.float32).tolist(), rng.permutation(6)[:6].tolist())
        return table[key]

    def expand(items):
        rows = [lp_of(c, n.words()) for c, n in items]
        return [r[0][:3] for r in rows], [r[1][:3] for r in rows]

    got = beam_search(expand, 3, 0, 5, 3, 2)
    for clip in range(3):
        def logprobs_of(words, clip=clip):
            v, i = lp_of(clip, words)
            out = torch.full((6,), -1e9)
            out[torch.tensor(i)] = torch.tensor(v)
            return out
        assert O.beam_decode_one(logprobs_of, 0, 5, 3, 2) == got[2 * clip:2 * clip + 2]


def test_caption_samples_dry_run(tmp_path):
    fakes = tmp_path / "fakes"
    fakes.mkdir()
    for stem in ("Y1", "Y2"):
        for j in range(2):
            np.save(fakes / f"{stem}_mel_sample_{j}.npy", np.zeros((80, 848), np.float32))
    csv = tmp_path / "val.csv"
    csv.write_text("audiocap_id,youtube_id,start_time,caption,file_name\n" +
                   "".join(f"{i},x,0,a cat {k},{stem}.wav\n" for i, (stem, k) in enumerate([(s, k) for s in ("Y1", "Y2") for k in range(5)])))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "caption_samples.py"), "--fakes", str(fakes), "--captions", str(csv), "--ckpt", "x",
                        "--vocab", "x", "--out", str(tmp_path / "out"), "--dry-run"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["clips"] == 4 and line["captions_per_clip"] == 5


def test_caption_kernels_no_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.access(nvcc, os.X_OK):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Iinclude", "-Itext-to-sound-synthesis_b200/csrc",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", "text-to-sound-synthesis_b200/csrc/caption.cu", "-o", os.devnull],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    entries = r.stderr.count("Compiling entry function")
    assert entries == 6
    assert r.stderr.count("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") == entries
    assert "lmem" not in r.stderr


def test_caption_words_follow_eval_py():
    """eval.py: <sos> dropped; a row without <eos> loses its last word to eos_ind; the caption stops at the first <eos>."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from caption_samples import words_of
    words = ["<sos>", "a", "dog", "<eos>", "barks"]
    assert words_of([0, 1, 2, 3, 4, 4], words, 3) == "a dog"
    assert words_of([0, 1, 2, 4], words, 3) == "a dog"          # no <eos>: the last word is overwritten
    assert words_of([0, 3, 3, 3], words, 3) == ""
    assert words_of([0], words, 3) == ""
