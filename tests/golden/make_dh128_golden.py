"""Generate tests/golden/gen_small_dh128.npz by running the UNMODIFIED reference with 128-wide attention heads.

Run in the build container only (needs /root/reference):   python tests/golden/make_dh128_golden.py
Built like make_golden.py (same stand-ins for the reference's third-party packages, same hash-keyed weights from oracle/synth.py): a
MaskGitTransformer with dim 256, 2 heads of dim_head = 128, depth 2, over an 8-token text context (not a multiple of 32), for
  - Transformer.forward: the conditional embeddings and the CFG logits on fixed ids;
  - MaskGit.generate at seq 16 (4 x 4 fmap, 6 steps) under torch.manual_seed noise;
  - the super-resolution generate at seq 64 (8 x 8 fmap, 16 conditioning tokens, 8 steps).
"""
import os
import sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import transformers  # noqa: F401  (must be imported BEFORE the accelerate stand-in is visible)
from transformers import T5Config

sys.path.insert(0, os.path.join(HERE, "_shims"))
sys.path.insert(0, "/root/reference")

from muse_maskgit_pytorch import t5 as ref_t5                      # noqa: E402
from muse_maskgit_pytorch import VQGanVAE, MaskGitTransformer, MaskGit   # noqa: E402

from oracle import synth, shapes                                    # noqa: E402

torch.set_grad_enabled(False)
ref_t5.T5_CONFIGS["synth-128"] = dict(config=T5Config(d_model=128))
DIM, HEADS, DH, DEPTH = 256, 2, 128, 2


def fill(module, table, seed):
    sd = module.state_dict()
    got = {k: tuple(v.shape) for k, v in sd.items() if not k.startswith("discr.") and k != "quantizer.mask"}
    assert got == {k: tuple(v) for k, v in table.items()}, sorted(set(got) ^ set(table))
    for k, v in synth.fill_state_dict(table, seed=seed).items():
        sd[k].copy_(torch.from_numpy(v))


def text_embeds(name, b, m, d, seed):
    te = torch.from_numpy(synth.normal(name, (b, m, d), seed))
    te[1::2, (3 * m) // 4:] = 0.
    return te


def transformer(seq_len, seed):
    tr = MaskGitTransformer(num_tokens=1024, dim=DIM, seq_len=seq_len, depth=DEPTH, dim_head=DH, heads=HEADS, t5_name="synth-128",
                            flash=False).eval()
    fill(tr, shapes.transformer_shapes(1024, DIM, seq_len, DEPTH, heads=HEADS, dim_head=DH, text_dim=128), seed=seed)
    return tr


def run_generate(mg, seed, **kw):
    torch.manual_seed(seed)
    g = {}
    orig = mg.vae.decode_from_ids
    mg.vae.decode_from_ids = lambda ids_, _o=orig: (g.__setitem__("ids", ids_.clone()), _o(ids_))[1]
    images = mg.generate(texts=["a"] * kw.pop("b"), cond_scale=3., temperature=1., **kw)
    mg.vae.decode_from_ids = orig
    return images, g["ids"]


vae_s = VQGanVAE(dim=16, layers=2, codebook_size=1024).eval()
fill(vae_s, shapes.vae_shapes(16, layers=2, codebook_size=1024), seed=12)
te = text_embeds("g4.te", 3, 8, 128, 14)

tr = transformer(16, seed=41)
ids = torch.from_numpy((synth.uniform("dh128.ids", (3, 16), 41) * 1025).astype(np.int64))
ids[:, ::3] = 1024
_, embed = tr(ids, text_embeds=te, return_embed=True)
cfg = tr.forward_with_cond_scale(ids, text_embeds=te, cond_scale=3.)

tr.encode_text = lambda texts: te
mg = MaskGit(image_size=16, transformer=tr, vae=vae_s).eval()
images, gen_ids = run_generate(mg, 790, b=3, timesteps=6)

tr2 = transformer(64, seed=42)
tr2.encode_text = lambda texts: te[:2]
mg2 = MaskGit(image_size=32, transformer=tr2, vae=vae_s, cond_image_size=16).eval()
cond = torch.from_numpy(synth.uniform("g5.cond", (2, 3, 16, 16), 15))
sr_images, sr_ids = run_generate(mg2, 791, b=2, cond_images=cond, timesteps=8)

out = dict(ids=ids, embed=embed, logits_cfg=cfg, images=images, gen_ids=gen_ids, sr_images=sr_images, sr_ids=sr_ids,
           u_probe=(torch.manual_seed(790), torch.zeros(7).uniform_(0, 1))[1])
np.savez_compressed(os.path.join(HERE, "gen_small_dh128.npz"), **{k: v.numpy() for k, v in out.items()})
print({k: tuple(v.shape) for k, v in out.items()})
