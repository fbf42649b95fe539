"""Seeded training batches as the DataLoader collates them from INTEGRATION.md's worker dict (the decoded images and
background frames, the object tables, the worker's augmentation draws), for build_ffb6d_train_item and
GraphedFrameTrainStep; and that document's trainer composition written out by hand."""
import numpy as np
import torch

import ffb6d_b200 as F
from ffb6d_b200 import augment as A
from ffb6d_b200.item import pose_gt_objects
from ffb6d_b200.synthetic import INTRINSICS, make_aug_frame, make_item_frame

CAM_SCALE = {"ycb": 10000.0, "linemod": 1000.0}
K_OF = {"ycb": INTRINSICS["ycb_K1"], "linemod": INTRINSICS["linemod"]}
IDENTITY_JITTER = np.array([0, 1, 2, 3, 1.0, 1.0, 1.0, 0.0])


def make_train_batch(seed, dataset, B, h, w, n_cls, n_kps=8, per_frame_K=False, device="cuda"):
    """``B`` frames mixing augmented and plain frames, jittered and plain frames and, among the augmented ones,
    ``apply_rgb`` both ways.  Images and object tables are CUDA tensors; the draws are host tensors."""
    rs = np.random.RandomState(seed)
    gen = torch.Generator().manual_seed(seed)
    ycb = dataset == "ycb"
    cls = tuple(range(1, min(n_cls, 4)))
    fr = [make_item_frame(seed * 31 + i, h=h, w=w, dataset=dataset, n_kps=n_kps, cls_ids=cls if ycb else (1,),
                          blobs=cls if ycb else (1,)) for i in range(B)]
    bk = [make_aug_frame(seed * 37 + i, h=h, w=w, dataset=dataset) for i in range(B)]
    objs = [pose_gt_objects(f["poses"], f["cls_ids"] if ycb else [1], f["kps"], f["ctrs"], 4 if ycb else 2, n_kps,
                            dataset=dataset) for f in fr]
    jitter, jittered, plans, augment, apply_rgb = [], [], [], [], []
    for i in range(B):
        on = (i + seed) % 2 == 0
        jitter.append(A.draw_color_jitter(1, gen)[0] if on else IDENTITY_JITTER)
        jittered.append(on)
        if (i + seed) % 3 != 2:
            aug = A.draw_frame_augmentation(rs, dataset, 5, rnd_typ="render")
            aug["apply_rgb"] = (i + seed) % 4 != 0
        else:
            aug = dict(plans=np.stack([A.identity_record(dataset, 0), A.identity_record(dataset, 1)]), augment=False,
                       apply_rgb=False)
        plans.append(aug["plans"])
        augment.append(aug["augment"])
        apply_rgb.append(aug["apply_rgb"])
    dev = torch.device(device)
    batch = {"dpt": np.stack([f["raw"] for f in fr]), "rgb": np.stack([f["rgb"] for f in fr]),
             "labels": np.stack([f["labels"] for f in fr]), "nrm_map": np.stack([f["nrm"] for f in fr]),
             "back_rgb": np.stack([b["back_rgb"] for b in bk]), "back_labels": np.stack([b["back_labels"] for b in bk]),
             "back_dpt": np.stack([b["back_dpt"] for b in bk])}
    batch.update({k: np.stack([o[k] for o in objs]) for k in objs[0]})
    batch = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in batch.items()}
    if per_frame_K:
        names = ("ycb_K1", "ycb_K2") if ycb else ("linemod", "ycb_K2")
        batch["K"] = torch.from_numpy(np.stack([INTRINSICS[names[i % 2]] for i in range(B)])).to(dev)
    batch.update(jitter=torch.from_numpy(np.stack(jitter)), jittered=torch.tensor(jittered),
                 plans=torch.from_numpy(np.stack(plans)), augment=torch.tensor(augment),
                 apply_rgb=torch.tensor(apply_rgb))
    return batch


def integration_item(batch, dataset, K, n_points, seed):
    """INTEGRATION.md's trainer lines, as a user writes them."""
    rgb = F.color_jitter(batch["rgb"], batch["jitter"].numpy(), active=batch["jittered"])
    rgb = F.rgb_add_noise(rgb, batch["plans"][:, 0].numpy(), seed=seed)
    rgb, dpt = F.add_real_back(rgb, batch["labels"], batch["dpt"], batch["back_rgb"], batch["back_labels"],
                               batch["back_dpt"], batch["apply_rgb"], dataset, active=batch["augment"])
    rgb = F.rgb_add_noise(rgb, batch["plans"][:, 1].numpy(), seed=seed)
    K = batch["K"].cpu().numpy() if "K" in batch else K
    item = F.build_ffb6d_item(dpt, CAM_SCALE[dataset], K, rgb, batch["labels"], batch["nrm_map"], batch, n_points,
                              seed=seed, fill=dataset == "ycb")
    item["rgb"] = item["rgb"].float()
    return item
