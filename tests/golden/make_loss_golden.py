"""Generate tests/golden/loss_small.npz: MaskGit.forward (the training loss, muse_maskgit_pytorch.py:623-741) of the UNMODIFIED reference
on the G4 / G5 / G6-G8 models of make_golden.py (same hash-generated weights and text embeddings).

Run in the build container only (needs /root/reference):   python tests/golden/make_loss_golden.py
Each case runs under torch.manual_seed(seed) + random.seed(py_seed) on the CPU.  The stored arrays are the case's input (token ids or images,
and the conditioning images of the super-resolution case), its seeds, keyword arguments, the values the reference's python random() calls
returned (`py_draws`) and the loss; tests/test_maskgit_loss_oracle.py replays every case through tests/loss_oracle.py, and
tests/test_gpu_maskgit_loss.py through MaskGit.forward.  The python draws are recorded rather than re-derived from py_seed because the
reference's @beartype wrapper of MaskGit.forward takes a getrandbits() from the same global generator on entry.
"""
import json
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import transformers  # noqa: F401,E402  (must be imported BEFORE the accelerate stand-in is visible)
from transformers import T5Config  # noqa: E402

sys.path.insert(0, os.path.join(HERE, "_shims"))
sys.path.insert(0, "/root/reference")

from muse_maskgit_pytorch import t5 as ref_t5                                    # noqa: E402
from muse_maskgit_pytorch import VQGanVAE, MaskGitTransformer, MaskGit, TokenCritic  # noqa: E402
import muse_maskgit_pytorch.muse_maskgit_pytorch as ref_module                     # noqa: E402

from oracle import synth, shapes                                                  # noqa: E402

torch.set_grad_enabled(False)


def fill(module, table, seed):
    sd = module.state_dict()
    for k, v in synth.fill_state_dict(table, seed=seed).items():
        sd[k].copy_(torch.from_numpy(v))


def text_embeds(name, b, m, d, seed):
    te = torch.from_numpy(synth.normal(name, (b, m, d), seed))
    te[1::2, (3 * m) // 4:] = 0.
    return te


ref_t5.T5_CONFIGS["synth-128"] = dict(config=T5Config(d_model=128))
te = text_embeds("g4.te", 3, 8, 128, 14)
vae = VQGanVAE(dim=16, layers=2, codebook_size=1024).eval()
fill(vae, shapes.vae_shapes(16, layers=2, codebook_size=1024), seed=12)


def transformer(seq_len, seed, **kw):
    tr = MaskGitTransformer(num_tokens=1024, dim=128, seq_len=seq_len, depth=2, dim_head=64, heads=2, t5_name="synth-128", flash=False, **kw)
    fill(tr, shapes.transformer_shapes(1024, 128, seq_len, 2, heads=2, text_dim=128), seed=seed)
    tr.encode_text = lambda texts: te[:len(texts)]
    return tr.eval()


tr = transformer(16, 13)                                  # G4
tr_sr = transformer(64, 15)                               # G5
tr_sc = transformer(16, 21, self_cond=True)               # G6 / G8
critic = TokenCritic(num_tokens=1024, dim=128, seq_len=16, depth=1, dim_head=64, heads=2, t5_name="synth-128", flash=False).eval()
fill(critic, shapes.transformer_shapes(1024, 128, 16, 1, heads=2, text_dim=128, add_mask_id=False, dim_out=1), seed=22)   # G7
critic.encode_text = lambda texts: te[:len(texts)]

models = dict(
    g4=lambda **kw: MaskGit(image_size=16, transformer=tr, vae=vae, **kw),
    g5=lambda **kw: MaskGit(image_size=32, transformer=tr_sr, vae=vae, cond_image_size=16, **kw),
    g6=lambda **kw: MaskGit(image_size=16, transformer=tr_sc, vae=vae, **kw),
    g7=lambda **kw: MaskGit(image_size=16, transformer=tr, vae=vae, token_critic=critic, **kw),
)


def g8(**kw):
    mg = MaskGit(image_size=16, transformer=tr_sc, vae=vae, self_token_critic=True, **kw)
    mg.token_critic.to_pred.weight.copy_(torch.from_numpy(synth.normal("g8.to_pred.weight", (1, 128), 23)) * 0.2)
    mg.token_critic.to_pred.bias.copy_(torch.from_numpy(synth.normal("g8.to_pred.bias", (1,), 23)) * 0.2)
    return mg


models["g8"] = g8

img16 = torch.from_numpy(synth.uniform("loss.img16", (3, 3, 16, 16), 40))
img32 = torch.from_numpy(synth.uniform("loss.img32", (2, 3, 32, 32), 41))
cond16 = torch.from_numpy(synth.uniform("g5.cond", (2, 3, 16, 16), 15))
ids16 = torch.from_numpy((synth.uniform("loss.ids", (3, 4, 4), 42) * 1024).astype(np.int64))

# name: (model, model kwargs, input, forward kwargs, torch seed, python seed)
CASES = dict(
    plain=("g4", {}, img16, {}, 800, 0),
    drop0=("g4", {}, img16, dict(cond_drop_prob=0.), 801, 1),
    drop1=("g4", {}, img16, dict(cond_drop_prob=1.), 802, 2),
    no_mask_token=("g4", dict(no_mask_token_prob=0.3), img16, {}, 803, 3),
    ids=("g4", {}, ids16, {}, 804, 4),
    selfcond=("g6", {}, img16, {}, 805, 0),                  # random.seed(0): first random() = 0.84 < self_cond_prob 0.9
    token_critic=("g7", {}, img16, {}, 806, 6),
    token_critic_temp=("g7", dict(critic_loss_weight=0.5), img16, dict(sample_temperature=0.7), 807, 7),
    self_critic=("g8", {}, img16, {}, 808, 0),
    superres=("g5", {}, img32, dict(cond_images=cond16), 809, 9),
)

py_draws = []
ref_random = ref_module.random
ref_module.random = lambda: (lambda v: (py_draws.append(v), v)[1])(ref_random())     # records, does not change the stream

out = {}
for name, (model, mkw, inp, fkw, seed, py_seed) in CASES.items():
    mg = models[model](**mkw).eval()
    torch.manual_seed(seed)
    random.seed(py_seed)
    py_draws.clear()
    # text_embeds, not texts: beartype checks a List[str] argument by sampling one of its items from python's global `random`, which would
    # move the reference's own random() draws
    loss = mg(inp, text_embeds=te[:inp.shape[0]], **fkw)
    out[f"{name}.loss"] = loss.reshape(1)
    out[f"{name}.input"] = inp
    out[f"{name}.seeds"] = torch.tensor([seed, py_seed])
    out[f"{name}.py_draws"] = torch.tensor(py_draws, dtype=torch.float64)
    if "cond_images" in fkw:
        out[f"{name}.cond_images"] = fkw["cond_images"]
    out[f"{name}.meta"] = np.frombuffer(json.dumps(dict(model=model, model_kw=mkw, kw={k: v for k, v in fkw.items() if k != "cond_images"})).encode(),
                                        dtype=np.uint8)
    print(name, float(loss))

np.savez_compressed(os.path.join(HERE, "loss_small.npz"), **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
