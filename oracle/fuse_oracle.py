"""LineMOD's `fuse` frames restated in numpy (DESIGN.md §4.34): the crop rule of ``FuseCropTable`` and the paste rule
of the header's ``ffb6d_fuse_rgbd``.

The paste is written as a painter's algorithm (each slot in order, its silhouette pixels overwriting what is there),
the kernel as a gather (each pixel takes the highest slot that holds it).  The two agree by construction of the rule,
and computing the frame's window of each crop with Python integers keeps every offset, however extreme, exact.
"""
import numpy as np


def crop_box(mask):
    """The inclusive bounding box ``(row0, row1, col0, col1)`` of ``mask != 0``, or None when it is empty."""
    sil = np.asarray(mask) != 0
    rows, cols = np.flatnonzero(sil.any(1)), np.flatnonzero(sil.any(0))
    if rows.size == 0:
        return None
    return int(rows[0]), int(rows[-1]), int(cols[0]), int(cols[-1])


def crop_frame(rgb, dpt, mask):
    """A decoded frame's crop: ``(rgb [h,w,3] uint8, dpt [h,w] uint16, sil [h,w] uint8 0/1, (row0, col0))``."""
    r0, r1, c0, c1 = crop_box(mask)
    win = (slice(r0, r1 + 1), slice(c0, c1 + 1))
    return (np.asarray(rgb)[win].copy(), np.asarray(dpt)[win].copy(),
            (np.asarray(mask)[win] != 0).astype(np.uint8), (r0, c0))


def fuse(crops, crop, offset, label, H, W, active=None, out=None):
    """Paste ``crops`` (a list of ``(rgb, dpt, sil)``) into ``B`` frames of ``H x W``.

    :param crop: ``[B,M]`` crop indices (outside ``[0, len(crops))``: nothing); :param offset: ``[B,M,2]`` (row, col)
      of each crop's top-left corner, any integers; :param label: ``[B,M]`` the slots' label values
    :param active: ``[B]`` bools or None; an inactive frame is not written
    :param out: None (zeros) or ``(dpt_mm [B,H,W] uint16, rgb [B,H,W,3] uint8, labels [B,H,W] uint8)``, copied
    :return: ``(dpt_mm, rgb, labels)``
    """
    crop, offset, label = np.asarray(crop), np.asarray(offset), np.asarray(label)
    B, M = crop.shape
    if out is None:
        dpt_o = np.zeros((B, H, W), np.uint16)
        rgb_o = np.zeros((B, H, W, 3), np.uint8)
        lab_o = np.zeros((B, H, W), np.uint8)
    else:
        dpt_o, rgb_o, lab_o = (np.array(t, copy=True) for t in out)
    for b in range(B):
        if active is not None and not active[b]:
            continue
        for s in range(M):
            k = int(crop[b, s])
            if not 0 <= k < len(crops):
                continue
            c_rgb, c_dpt, c_sil = crops[k]
            h, w = c_sil.shape
            row, col = int(offset[b, s, 0]), int(offset[b, s, 1])
            # the frame window the crop covers, and the same window in crop coordinates
            fr0, fr1 = max(row, 0), min(row + h, H)
            fc0, fc1 = max(col, 0), min(col + w, W)
            if fr0 >= fr1 or fc0 >= fc1:
                continue
            win = (slice(fr0 - row, fr1 - row), slice(fc0 - col, fc1 - col))
            on = c_sil[win] != 0
            dpt_o[b, fr0:fr1, fc0:fc1][on] = c_dpt[win][on]
            rgb_o[b, fr0:fr1, fc0:fc1][on] = c_rgb[win][on]
            lab_o[b, fr0:fr1, fc0:fc1][on] = label[b, s]
    return dpt_o, rgb_o, lab_o
