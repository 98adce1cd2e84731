"""CPU oracle of MaskGit.extrapolate's token loop: an fp32 restatement on torch CPU, composed from tests/inpaint_oracle.inpaint_ids.  The reference
has no extrapolation; the loop restated here is:

  canvas = ids0 at the kept side, mask_id elsewhere; K = amount / (stride * p) windows of f x f tokens
  window w: the block whose far edge lies stride * (w + 1) tokens past the input's edge; known = the canvas block, regen = its `stride`
  columns (rows) at the far side; inpaint_ids with the noise of its step s drawn as noise_fn(w * timesteps + s, shape); the strip of the
  result is written into the canvas."""
import torch

from tests import inpaint_oracle as IO

DIRECTIONS = ("right", "left", "down", "up")


def plan(direction, in_h, in_w, f, stride, K):
    """(canvas (h, w), input corner (row, col), [K] window corners (row, col)) in tokens for an input of in_h x in_w tokens."""
    assert direction in DIRECTIONS
    grow = K * stride
    if direction in ("right", "left"):
        assert in_h == f and in_w >= f
        canvas = (f, in_w + grow)
        if direction == "right":
            return canvas, (0, 0), [(0, in_w + stride * (w + 1) - f) for w in range(K)]
        return canvas, (0, grow), [(0, grow - stride * (w + 1)) for w in range(K)]
    assert in_w == f and in_h >= f
    canvas = (in_h + grow, f)
    if direction == "down":
        return canvas, (0, 0), [(in_h + stride * (w + 1) - f, 0) for w in range(K)]
    return canvas, (grow, 0), [(grow - stride * (w + 1), 0) for w in range(K)]


def strip(direction, f, stride):
    """(f, f) bool: the tokens a window generates."""
    s = torch.zeros((f, f), dtype=torch.bool)
    if direction == "right":
        s[:, f - stride:] = True
    elif direction == "left":
        s[:, :stride] = True
    elif direction == "down":
        s[f - stride:, :] = True
    else:
        s[:stride, :] = True
    return s


def initial_canvas(ids0, direction, f, stride, K, mask_id):
    """(b, H, W) int64: ids0 (b, in_h, in_w) placed at the kept side of the canvas, mask_id elsewhere."""
    b, in_h, in_w = ids0.shape
    (H, W), (r, c), _ = plan(direction, in_h, in_w, f, stride, K)
    canvas = torch.full((b, H, W), mask_id, dtype=torch.long)
    canvas[:, r:r + in_h, c:c + in_w] = ids0
    return canvas


def extrapolate_ids(sd, cfg, text_embeds, ids0, direction, K, stride, mask_id, noise_fn, timesteps=18, trace=None, **kw):
    """ids0 (b, in_h, in_w) int64: the encoded image tokens.  Returns the (b, H, W) canvas.  noise_fn as in inpaint_ids; kw goes to inpaint_ids
    (cond_scale, temperature, critic, ...).  trace (list) receives one dict per window: corner, known (b, f*f), ids (b, f*f) after it."""
    b = ids0.shape[0]
    f = _fmap(sd)
    canvas = initial_canvas(ids0, direction, f, stride, K, mask_id)
    _, _, corners = plan(direction, ids0.shape[1], ids0.shape[2], f, stride, K)
    regen = strip(direction, f, stride).reshape(1, -1).expand(b, -1)
    for w, (r, c) in enumerate(corners):
        known = canvas[:, r:r + f, c:c + f].reshape(b, -1).clone()
        ids = IO.inpaint_ids(sd, cfg, text_embeds, known, regen, mask_id, lambda s, shape, w=w: noise_fn(w * timesteps + s, shape),
                             timesteps=timesteps, **kw)
        block = canvas[:, r:r + f, c:c + f]
        block[regen.reshape(b, f, f)] = ids.reshape(b, f, f)[regen.reshape(b, f, f)]
        if trace is not None:
            trace.append(dict(corner=(r, c), known=known, ids=ids))
    return canvas


def _fmap(sd):
    """f of the transformer state dict: its positional embedding holds f * f rows."""
    key = next(k for k in sd if k.endswith("pos_emb.weight"))
    n = sd[key].shape[0]
    f = int(round(n ** 0.5))
    assert f * f == n, n
    return f
