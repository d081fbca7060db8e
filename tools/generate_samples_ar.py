"""Caption file -> .npy mels + .wav clips from the autoregressive SpecVQGAN transformer (Codebook/configs/caps_transformer*.yaml) on the H100
kernels: the flow of Codebook/evaluation/generate_samples_caps.py with the condition computed from the caption, as
Codebook/generete_text_fea/generate_fea_clip.py does it (CLIP ViT-B/32 `encode_text`: the pooled, projected feature of the end token).

    python tools/generate_samples_ar.py --config caps_transformer.yaml --ckpt last.ckpt --clip-ckpt ViT-B-32.pt --vocoder-ckpt best_netG.pt \\
        --captions val.csv --out samples/ [--batch-size 96] [--temperature 1.0] [--top-k 100] [--greedy] [--no-condition] [--bpe vocab.txt.gz]

Defaults are Codebook/evaluation/configs/sampler.yaml's: batch 96, temperature 1.0, top_k 100, sampled (sample_next_tok_from_pred_dist), 'nopix'
(all 265 tokens generated; 'half' needs ground-truth mels and is not offered from captions).  --no-condition is the sampler's `no_condition`: the
transformer sees a zero feature.  The YAML is the reference's own file; its `target:` strings are rewritten to this package.  Captions come
from a CSV with `file_name,caption` columns; each caption gives one clip `{file}_mel_sample_{n}` (n counts captions of the same file), written in
the layout Codebook/evaluate.py reads (pipeline.save_clip).  --dry-run builds everything on the CPU and stops before the first kernel."""
import argparse
import os
import sys

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200 import pipeline  # noqa: E402
from diffsound_b200.modeling.codecs.text_codec.tokenize import tokenize  # noqa: E402
from diffsound_b200.modeling.embeddings.clip_text_embedding import CLIPTextEmbedding  # noqa: E402
from diffsound_b200.modeling.modules.clip.simple_tokenizer import SimpleTokenizer  # noqa: E402
from diffsound_b200.utils.misc import instantiate_from_config, retarget_config  # noqa: E402
from diffsound_b200.vocoder.modules import Generator  # noqa: E402
from tools.generate_samples import read_captions  # noqa: E402

GRID = (5, 53)  # mel 80 x 848 -> 5 x 53 codes (caps_transformer.yaml's permuter)


def build(args):
    with open(args.config) as f:
        cfg = retarget_config(yaml.full_load(f)["model"])
    p = cfg["params"]
    p["first_stage_config"]["params"]["ckpt_path"] = args.codec_ckpt  # the YAML's path is the authors' machine
    p["first_stage_config"]["params"]["lossconfig"] = None
    p.pop("ckpt_path", None)
    model = instantiate_from_config(cfg)
    if args.ckpt:
        sd = torch.load(args.ckpt, map_location="cpu")
        missing, unexpected = model.load_state_dict(sd.get("state_dict", sd), strict=False)  # generate_samples_caps.py:138-141
        print(f"model: {len(missing)} missing / {len(unexpected)} unexpected keys")
    text = CLIPTextEmbedding(pick_last_embedding=True, normalize=False, clip_ckpt_path=args.clip_ckpt)
    vocoder = None
    if args.vocoder_ckpt:
        vocoder = Generator(80, 32, 3)
        vocoder.load_state_dict(torch.load(args.vocoder_ckpt, map_location="cpu"))
    return model, text, SimpleTokenizer(bpe_path=args.bpe), vocoder


@torch.no_grad()
def caption_features(text_model, tokenizer, captions):
    """generate_fea_clip.py:12-25: clip.tokenize -> encode_text, the (B, 512) pooled feature, as the (B, 512, 1) RawFeatsStage input."""
    tok = tokenize(captions, context_length=77, add_start_and_end=True, with_mask=False, tokenizer=tokenizer)["token"]
    return text_model.encode_text(tok.to(text_model.text_projection.device)).float().unsqueeze(-1)


@torch.no_grad()
def synthesize(model, vocoder, feats, *, temperature=1.0, top_k=100, sample=True, no_condition=False):
    """feats (B, 512, 1) -> dict(tokens (B, 265), mel (B, 1, 80, 848), wav (B, 1, T) or None): sample_spectrogram (generate_samples_caps.py:169-229)
    in 'nopix' mode, then decode_to_img and the MelGAN vocoder on (mel + 1) / 2."""
    c = torch.zeros_like(feats) if no_condition else feats
    _, c = model.encode_to_c(c)
    B = c.shape[0]
    x0 = torch.zeros(B, 0, dtype=torch.long, device=c.device)
    ids, _ = model.sample(x0, c, GRID[0] * GRID[1], temperature=temperature, sample=sample, top_k=top_k)
    emb = model.first_stage_model.quantize.embedding.weight.shape[1]
    mel = model.decode_to_img(ids, (B, emb, GRID[0], GRID[1]))
    wav = vocoder((mel[:, 0] + 1) / 2) if vocoder is not None else None
    return {"tokens": ids, "mel": mel, "wav": wav}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--config", required=True, help="Codebook/configs/caps_transformer*.yaml")
    ap.add_argument("--ckpt", default=None, help="Lightning checkpoint of the transformer ({'state_dict': ...})")
    ap.add_argument("--codec-ckpt", default=None, help="SpecVQGAN Lightning checkpoint (only needed if --ckpt does not hold first_stage_model.*)")
    ap.add_argument("--clip-ckpt", default=None, help="OpenAI CLIP ViT-B/32 weights (state_dict or TorchScript archive)")
    ap.add_argument("--bpe", default=None, help="bpe_simple_vocab_16e6.txt.gz (default: $DIFFSOUND_BPE_VOCAB or the reference checkout)")
    ap.add_argument("--vocoder-ckpt", default=None, help="MelGAN generator state_dict")
    ap.add_argument("--captions", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch-size", type=int, default=96)
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--top-k", type=int, default=100, help="0 = no truncation")
    ap.add_argument("--greedy", action="store_true", help="argmax instead of sampling (sample_next_tok_from_pred_dist: False)")
    ap.add_argument("--no-condition", action="store_true")
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--dry-run", action="store_true")
    a = ap.parse_args(argv)
    model, text, tokenizer, vocoder = build(a)
    caps = read_captions(a.captions)
    jobs = [(name.split(".")[0], n, t) for name, texts in caps.items() for n, t in enumerate(texts)]
    print(f"{len(caps)} files, {len(jobs)} captions, temperature {a.temperature}, top_k {a.top_k or None}, "
          f"{'greedy' if a.greedy else 'sampled'}, {'no condition' if a.no_condition else 'CLIP condition'}")
    if a.dry_run:
        return model, text, vocoder, jobs
    model, text = model.cuda().eval(), text.cuda()
    vocoder = vocoder.cuda().eval() if vocoder is not None else None
    torch.manual_seed(a.seed)
    for i in range(0, len(jobs), a.batch_size):
        chunk = jobs[i:i + a.batch_size]
        feats = caption_features(text, tokenizer, [t for _, _, t in chunk])
        out = synthesize(model, vocoder, feats, temperature=a.temperature, top_k=a.top_k or None, sample=not a.greedy, no_condition=a.no_condition)
        for j, (base, n, _) in enumerate(chunk):
            pipeline.save_clip(a.out, base, n, out["mel"][j], None if out["wav"] is None else out["wav"][j])
    return 0


if __name__ == "__main__":
    main()
