"""Melception feature extractor and evaluation metrics, CPU side: the oracle against the reference's own outputs, the drop-in's parameter tree
against the reference's key list, the metric restatements against the reference's numbers, and evaluate_samples.py's file listing / pairing."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.helpers import GOLD, ROOT

import _pkg

_pkg.load()

from oracle import melception_oracle as MO  # noqa: E402


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLD, "melception_ref.npz"))


def mel_input(seed, B, T):
    """Must stay identical to oracle/gen_golden_melception.py:mel_input (inputs are regenerated, not stored)."""
    rng = np.random.Generator(np.random.Philox(seed))
    return torch.from_numpy(rng.random(size=(B, 80, T), dtype=np.float32)) * 4 - 2


@pytest.mark.parametrize("tag", ["he", "wide"])
def test_oracle_reproduces_reference(ref, tag):
    seed, B, T, xseed = ref[f"{tag}.cfg"].tolist()
    sd = MO.make_melception_state_dict(seed, tag)
    np.testing.assert_array_equal(MO.state_dict_checksum(sd), ref[f"{tag}.sd_checksum"])
    feats = MO.melception_forward(sd, mel_input(xseed, B, T), MO.FEATURES, torch.float64)
    for name, f in zip(MO.FEATURES, feats):
        r = torch.from_numpy(ref[f"{tag}.{name}"]).double()
        assert f.shape == r.shape, (name, f.shape, r.shape)
        err = float((f - r).abs().max() / r.abs().max())
        assert err < 1e-5, (tag, name, err)


def test_oracle_early_exit_and_order():
    sd = MO.make_melception_state_dict(3, "he")
    x = mel_input(5, 1, 96)
    full = dict(zip(MO.FEATURES, MO.melception_forward(sd, x, MO.FEATURES)))
    for fl in (["64"], ["768", "64"], ["logits"], ["logits_unbiased"], ["2048", "logits", "192"]):
        got = MO.melception_forward(sd, x, fl)
        assert len(got) == len(fl)
        for name, g in zip(fl, got):
            torch.testing.assert_close(g, full[name], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("aux", [True, False])
def test_dropin_state_dict_matches_reference_keys(ref, tmp_path, aux):
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    sd = MO.make_melception_state_dict(0, "he", aux_logits=aux)
    path = str(tmp_path / "w.pt")
    torch.save({"model": sd}, path)
    m = Melception(309, ["logits_unbiased", "2048", "logits"], path, aux_logits=aux)
    tag = "keys_aux" if aux else "keys_noaux"
    assert list(m.state_dict()) == ref[tag].tolist()
    assert [",".join(map(str, v.shape)) for v in m.state_dict().values()] == ref[tag + "_shapes"].tolist()
    assert len(m.state_dict()) == (580 if aux else 566)
    assert all(not p.requires_grad for p in m.parameters())
    for k, v in sd.items():
        assert torch.equal(m.state_dict()[k], v), k
    assert m.convert_features_tuple_to_dict((1, 2, 3)) == {"logits_unbiased": 1, "2048": 2, "logits": 3}


def test_dropin_refuses_cpu_and_training(tmp_path):
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    path = str(tmp_path / "w.pt")
    torch.save({"model": MO.make_melception_state_dict(0, "he")}, path)
    m = Melception(309, ["2048"], path)
    with pytest.raises(RuntimeError, match="eval mode"):
        m.train()(torch.zeros(1, 80, 96))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(torch.zeros(1, 80, 96))
    with pytest.raises(RuntimeError):  # strict loading: a missing key is an error, as in the reference
        sd = MO.make_melception_state_dict(0, "he")
        sd.pop("fc.bias")
        torch.save({"model": sd}, path)
        Melception(309, ["2048"], path)


def metric_inputs():
    """Must stay identical to oracle/gen_golden_melception.py:metric_inputs."""
    rng = np.random.Generator(np.random.Philox(2024))
    keys = [f"Y{k:03d}abc_{k * 7 % 13}" for k in range(24)]
    real_names = [f"/reals/val/{k}_mel.npy" for k in keys]
    fake_names = [f"/fakes/caps_validation/cls_0/{k}_sample_{n}.npy" for k in keys for n in range(4)]
    r_logits = rng.random(size=(24, 20)) * 6 - 3
    f_logits = np.repeat(r_logits, 4, 0) + rng.random(size=(96, 20)) * 2 - 1
    r_feats = rng.random(size=(24, 32)) * 2
    f_feats = rng.random(size=(96, 32)) * 2 + 0.3
    f32 = lambda a: torch.from_numpy(a.astype(np.float32))
    return (fake_names, f32(f_logits), f32(f_feats)), (real_names, f32(r_logits), f32(r_feats))


def test_metrics_match_reference_numbers():
    from diffsound_b200.evaluation.metrics import fid, isc, kid, kl
    g = np.load(os.path.join(GOLD, "eval_metrics.npz"))
    want = dict(zip(g["names"].tolist(), g["values"].tolist()))
    (fn, fl, ff), (rn, rl, rf) = metric_inputs()
    d1 = {"file_path_": fn, "logits": fl, "logits_unbiased": fl - 0.5, "2048": ff}
    d2 = {"file_path_": rn, "logits": rl, "logits_unbiased": rl - 0.5, "2048": rf}
    got = {}
    got.update(kl.calculate_kl(d1, d2, "logits", "caps"))
    got.update(isc.calculate_isc(d1, "logits_unbiased", 2020, True, 10))
    got.update(fid.calculate_fid(d1, d2, "2048"))
    got.update(kid.calculate_kid(d1, d2, 100, 1000, 3, None, 1, 2020, "2048"))
    assert set(got) == set(want)
    assert got["kullback_leibler_divergence"] == want["kullback_leibler_divergence"]
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-10 * abs(want[k]), (k, got[k], want[k])
    with pytest.raises(NotImplementedError):
        kl.calculate_kl(d1, d2, "logits", "vggsound")


def test_evaluate_samples_dry_run_pairs_like_kl(tmp_path):
    fakes, reals = tmp_path / "fakes", tmp_path / "reals"
    keys = ["Yabc_1", "Y-def_7", "Yxyz_30"]
    for i, k in enumerate(keys):
        (reals / "val").mkdir(parents=True, exist_ok=True)
        np.save(reals / "val" / f"{k}_mel.npy", np.zeros((80, 8), np.float32))
        for n in range(2 + i):
            d = fakes / ("cls_1" if n % 2 else "cls_0")
            d.mkdir(parents=True, exist_ok=True)
            np.save(d / f"{k}_sample_{n}.npy", np.zeros((80, 8), np.float32))
    np.save(fakes / "stray_sample_0.npy", np.zeros(1))  # outside any class folder: ignored, as DatasetFolder does
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "evaluate_samples.py"), "--fakes", str(fakes), "--reals", str(reals), "--dry-run"],
                       capture_output=True, text=True, check=True)
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["n_reals"] == 3 and out["n_fakes"] == 9 and out["n_paired_fakes"] == 9
    names = [os.path.relpath(p, fakes) for p in out["fakes"]]
    assert names == sorted(names, key=lambda s: (s.split("/")[0], s.split("/")[1]))  # class folder first, then file name
    assert names[0].startswith("cls_0/") and names[-1].startswith("cls_1/")
    for k in keys:
        assert sorted(os.path.basename(p) for p in out["pairs"][k]) == [f"{k}_sample_{n}.npy" for n in range(2 + keys.index(k))]
