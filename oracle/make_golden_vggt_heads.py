"""ORACLE -- test infrastructure only (see oracle/README.md).  Writes tests/golden/vggt_point_track_mini.npz from the
reference's own VGGT modules (vggt/heads/dpt_head.py, track_head.py, track_modules/, models/vggt.py), run on the CPU
in float32 at a reduced size:

  heads_*  the point head (DPTHead output_dim 4, "inv_log") and the track head (TrackHead: 128-feature DPT extractor,
           tracker with 7 levels, 4 iterations) on seeded tokens, images and query points;
  model_*  the whole VGGT at a mini width (embed_dim 64, a 24-layer convolutional aggregator of one 64-wide head,
           every head enabled) called as model(images, query_points).

Weights are r3g.vggt_heads.random_state_dict(**WEIGHTS) loaded with strict=True into the reference modules, which also
pins the key names and shapes of the generated state dict; the inputs come from seeded generators (inputs()).  Only
the seeds, checksums of the inputs and the outputs are stored (the dense maps subsampled), so the file stays small.
Run: python oracle/make_golden_vggt_heads.py"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "3d-re-gen_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "vggt_point_track_mini.npz")
EMBED, LAYERS, S, H, W, NQ, ITERS = 64, 24, 2, 140, 154, 16, 4      # 140 / 2 = 70 >= 2^6: seven pyramid levels
WEIGHTS = dict(seed=11, embed_dim=EMBED, depth=LAYERS, vit_depth=0, trunk_depth=4, img_size=H, full=True,
               patch_embed="conv")
INPUT_SEED = 12
SUB = {"heads": 2, "model": 4}     # stride of the stored subsample of each dense map


def inputs():
    """(tokens: LAYERS x [1, S, 5 + P, 2 * EMBED], images [1, S, 3, H, W] in [0, 1], query points [1, NQ, 2] pixels)."""
    g = torch.Generator().manual_seed(INPUT_SEED)
    P = (H // 14) * (W // 14)
    toks = [torch.randn(1, S, 5 + P, 2 * EMBED, generator=g) for _ in range(LAYERS)]
    images = torch.rand(1, S, 3, H, W, generator=g)
    qp = torch.rand(1, NQ, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])
    return toks, images, qp


def checksum(t):
    return np.float64(t.double().abs().sum().item())


def main():
    import ref_import
    from r3g.vggt_heads import random_state_dict
    ref_import.vggt_package()
    from vggt.heads.dpt_head import DPTHead
    from vggt.heads.track_head import TrackHead
    from vggt.models.aggregator import Aggregator
    from vggt.models.vggt import VGGT

    sd = random_state_dict(**WEIGHTS)
    toks, images, qp = inputs()
    z = {"weights_seed": np.int64(WEIGHTS["seed"]), "input_seed": np.int64(INPUT_SEED),
         "cfg": np.array([EMBED, LAYERS, S, H, W, NQ, ITERS], np.int64),
         "sum_tokens": checksum(torch.stack(toks)), "sum_images": checksum(images), "sum_query": checksum(qp)}

    def sub(name, t, k):
        z[name] = t[..., ::k, ::k, :].numpy() if t.dim() == 5 else t[..., ::k, ::k].numpy()

    point = DPTHead(dim_in=2 * EMBED, output_dim=4, activation="inv_log", conf_activation="expp1").eval()
    point.load_state_dict({k[len("point_head."):]: v for k, v in sd.items() if k.startswith("point_head.")}, strict=True)
    track = TrackHead(dim_in=2 * EMBED, patch_size=14).eval()
    track.load_state_dict({k[len("track_head."):]: v for k, v in sd.items() if k.startswith("track_head.")}, strict=True)
    with torch.no_grad():
        pts, conf = point(toks, images=images, patch_start_idx=5)
        track_list, vis, tconf = track(toks, images=images, patch_start_idx=5, query_points=qp, iters=ITERS)
    sub("heads_points", pts, SUB["heads"])
    sub("heads_points_conf", conf, SUB["heads"])
    z["heads_track"] = torch.stack(track_list).numpy()
    z["heads_vis"], z["heads_conf"] = vis.numpy(), tconf.numpy()

    torch.manual_seed(0)
    model = VGGT(img_size=H, patch_size=14, embed_dim=EMBED).eval()
    model.aggregator = Aggregator(img_size=H, patch_size=14, embed_dim=EMBED, depth=LAYERS, num_heads=1,
                                  patch_embed="conv").eval()
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        pred = model(images[0], qp[0])
    z["model_keys"] = np.array(sorted(pred))
    for k, v in pred.items():
        if k == "pose_enc_list":
            z["model_pose_enc_list"] = torch.stack(v).numpy()
            continue
        z["model_shape_" + k] = np.array(v.shape, np.int64)
        if k in ("depth", "depth_conf", "world_points", "world_points_conf"):
            sub("model_" + k, v, SUB["model"])
        elif k != "images":
            z["model_" + k] = v.numpy()
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes;", {k: tuple(v.shape) for k, v in pred.items() if torch.is_tensor(v)})


if __name__ == "__main__":
    main()
