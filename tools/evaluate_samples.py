"""Score generated clips against real ones: KL, ISc, FID and KID from Melception features on the H100 -- the flow of the reference's
Codebook/evaluate.py with the caps config (evaluation/configs/eval_melception_caps.yaml), without omegaconf or the reference checkout.

    python tools/evaluate_samples.py --fakes samples/caps_validation --reals data/audiocaps/features/val \
        --weights melception.pt --stats train_means_stds_melspec_10s_22050hz.txt
    python tools/evaluate_samples.py --fakes ... --reals ... --dry-run      # list files and the fake -> real pairing; no GPU

Inputs are read as torchvision's DatasetFolder does (FakesFolder, evaluation/datasets/fakes.py:28-76): sorted class sub-folders of the root, then
sorted files ending in the extension ('.npy' fakes, '_mel.npy' reals); ISc's seeded shuffle depends on that order.  Each mel (80, T) is normalised
per mel bin with the (80, 2) mean / std text file (StandardNormalizeAudio), fused into the feature extractor's first kernel.  Prints one JSON line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CAPS = dict(num_classes=309, features_list=["logits_unbiased", "2048", "logits"], isc=dict(splits=10, samples_shuffle=True, rng_seed=2020),
            kid=dict(subsets=100, subset_size=1000, degree=3, gamma=None, coef0=1, rng_seed=2020))


def list_folder(root, ext):
    """Files under root in DatasetFolder order: sorted class directories, os.walk in sorted order inside each, sorted file names."""
    classes = sorted(e.name for e in os.scandir(root) if e.is_dir())
    if not classes:
        raise FileNotFoundError(f"{root}: no class sub-folder (the files must sit in at least one sub-directory, as for DatasetFolder)")
    out = []
    for c in classes:
        for r, _, names in sorted(os.walk(os.path.join(root, c), followlinks=True)):
            out += [os.path.join(r, n) for n in sorted(names) if n.lower().endswith(ext.lower())]
    if not out:
        raise FileNotFoundError(f"{root}: no file ending in {ext}")
    return out


def pairing(fakes, reals):
    """{real key: [fake paths]} as the caps KL pairs them (file stem without '_mel', cut at '_sample_')."""
    import _pkg
    _pkg.load()
    from diffsound_b200.evaluation.metrics.kl import path_to_sharedkey
    groups = {path_to_sharedkey(p, "caps"): [] for p in reals}
    for p in fakes:
        k = path_to_sharedkey(p, "caps")
        if k in groups:
            groups[k].append(p)
    return groups


def extract(model, paths, batch_size):
    import torch
    feats = {k: [] for k in model.features_list}
    n = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, len(paths), batch_size):
        x = torch.from_numpy(np.stack([np.load(p).astype(np.float32) for p in paths[i:i + batch_size]])).cuda()
        for k, v in model.convert_features_tuple_to_dict(model(x)).items():
            feats[k].append(v.cpu())
        n += x.shape[0]
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    out = {k: torch.cat(v, 0) for k, v in feats.items()}
    out["file_path_"] = list(paths)
    return out, n / dt


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--fakes", required=True, help="root of the generated mels (<root>/<class>/<key>_sample_<n>.npy)")
    ap.add_argument("--reals", required=True, help="root of the real mels (<root>/<class>/<key>_mel.npy)")
    ap.add_argument("--fakes-ext", default=".npy")
    ap.add_argument("--reals-ext", default="_mel.npy")
    ap.add_argument("--weights", help="Melception checkpoint {'model': state_dict}")
    ap.add_argument("--stats", help="(80, 2) text file of per-mel-bin mean / std (train_means_stds_*.txt)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--dry-run", action="store_true", help="list the files and the pairing, touch no GPU")
    a = ap.parse_args()
    fakes, reals = list_folder(a.fakes, a.fakes_ext), list_folder(a.reals, a.reals_ext)
    groups = pairing(fakes, reals)
    if a.dry_run:
        print(json.dumps({"fakes": fakes, "reals": reals, "pairs": {k: v for k, v in groups.items()},
                          "n_fakes": len(fakes), "n_reals": len(reals), "n_paired_fakes": sum(len(v) for v in groups.values())}))
        return
    if not a.weights or not a.stats:
        ap.error("--weights and --stats are needed unless --dry-run")
    import torch
    import _pkg
    _pkg.load()
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    from diffsound_b200.evaluation.metrics import fid, isc, kid, kl
    if not torch.cuda.is_available():
        raise SystemExit("feature extraction needs a CUDA device (no CPU path)")
    model = Melception(CAPS["num_classes"], CAPS["features_list"], a.weights).cuda().eval()
    means, stds = np.loadtxt(a.stats).T
    model.engine.set_normalization(means, stds)
    f1, r1 = extract(model, fakes, a.batch_size)
    f2, r2 = extract(model, reals, a.batch_size)
    out = {}
    out.update(kl.calculate_kl(f1, f2, "logits", "caps"))
    out.update(isc.calculate_isc(f1, "logits_unbiased", **CAPS["isc"]))
    out.update(fid.calculate_fid(f1, f2, "2048"))
    out.update(kid.calculate_kid(f1, f2, feat_layer_name="2048", **CAPS["kid"]))
    out.update(n_fakes=len(fakes), n_reals=len(reals), clips_per_s_fakes=round(r1, 2), clips_per_s_reals=round(r2, 2),
               gpu=torch.cuda.get_device_name())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
