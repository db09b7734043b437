"""Writes tests/golden/clip_bpe/{merges.txt, vocab.json}: the part of the CLIP BPE vocabulary (the files that ship in
the reference tree, swift/StableDiffusionTests/Resources) that the known-answer prompts of test_tokenizer.py touch.
Merges keep their relative order (BPE only compares ranks of pairs that can occur in these words); vocabulary entries
keep their ids.  Run where the reference tree is present:

    python tests/golden/make_golden_tokenizer.py /path/to/reference
"""
import json
import os
import re
import sys

PROMPTS = ["a photo of an astronaut riding a horse on mars", "Apple CoreML developer tools on a Macbook Air are fast"]


def main(ref_root):
    res = os.path.join(ref_root, "swift", "StableDiffusionTests", "Resources")
    words = {w + "</w>" for p in PROMPTS for w in re.findall(r"[a-z]+|[0-9]|[^\sa-z0-9]+", p.lower())}
    with open(os.path.join(res, "merges.txt"), encoding="utf-8") as f:
        lines = f.read().split("\n")
    kept = [lines[0]] + [ln for ln in lines[1:] if ln.count(" ") == 1 and any(ln.replace(" ", "") in w for w in words)]
    with open(os.path.join(res, "vocab.json"), encoding="utf-8") as f:
        vocab = json.load(f)
    sub = {t: i for t, i in vocab.items() if t.startswith("<|") or any(t in w for w in words)}
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "clip_bpe")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "merges.txt"), "w", encoding="utf-8") as f:
        f.write("\n".join(kept) + "\n")
    with open(os.path.join(out, "vocab.json"), "w", encoding="utf-8") as f:
        json.dump(sub, f, ensure_ascii=False, sort_keys=True, indent=0)


if __name__ == "__main__":
    main(sys.argv[1])
