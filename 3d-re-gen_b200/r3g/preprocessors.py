"""Host-side image preparation, interface of Hunyuan3D-2/hy3dgen/shapegen/preprocessors.py:30-159
(ImageProcessorV2): alpha-bbox recentre on a white square, cubic resize to `size`, scale to [-1, 1];
MVImageProcessorV2 does that per view of a multi-view dict and stacks the views in index order.
CPU / OpenCV work done once per object; not a kernel target (SURVEY.md section 8a row a1)."""
import cv2
import numpy as np
import torch
from PIL import Image


def array_to_tensor(np_array):
    """uint8 HxWxC -> float32 [1, C, H, W] in [-1, 1] (preprocessors.py:21-27)."""
    a = np.ascontiguousarray(np_array).astype(np.float32) / 255.0 * 2.0 - 1.0
    # channels-first in numpy: torch's strided permute().contiguous() of a [512,512,3] CPU tensor took 21 ms per call
    return torch.from_numpy(np.ascontiguousarray(a.transpose(2, 0, 1))[None])


class ImageProcessorV2:
    def __init__(self, size=512, border_ratio=None):
        self.size = size
        self.border_ratio = border_ratio

    @staticmethod
    def recenter(image, border_ratio=0.2):
        """preprocessors.py:36-88.  Returns (rgb uint8 [S,S,3] composited on white, alpha uint8 [S,S,1])."""
        if image.shape[-1] == 4:
            alpha = image[..., 3]
        else:
            alpha = np.full(image.shape[:2], 255, dtype=image.dtype)
            image = np.concatenate([image, alpha[..., None]], axis=-1)
        H, W, C = image.shape
        side = max(H, W)
        rows, cols = np.nonzero(alpha)
        r0, r1, c0, c1 = rows.min(), rows.max(), cols.min(), cols.max()
        bh, bw = r1 - r0, c1 - c0
        if bh == 0 or bw == 0:
            raise ValueError("input image is empty")
        target = int(side * (1 - border_ratio))
        s = target / max(bh, bw)
        nh, nw = int(bh * s), int(bw * s)
        top, left = (side - nh) // 2, (side - nw) // 2
        canvas = np.zeros((side, side, C), dtype=np.uint8)
        # note: the reference crops [min:max) (exclusive of the last row/column) -- replicated
        canvas[top:top + nh, left:left + nw] = cv2.resize(image[r0:r1, c0:c1], (nw, nh), interpolation=cv2.INTER_AREA)
        a = canvas[..., 3:].astype(np.float32) / 255
        rgb = canvas[..., :3] * a + 255.0 * (1 - a)
        return rgb.clip(0, 255).astype(np.uint8), (a * 255).clip(0, 255).astype(np.uint8)

    def load_image(self, image, border_ratio=0.15, to_tensor=True):
        if isinstance(image, str):
            arr = cv2.imread(image, cv2.IMREAD_UNCHANGED)
            rgb, mask = self.recenter(arr, border_ratio=border_ratio)
            rgb = cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB)
        elif isinstance(image, Image.Image):
            rgb, mask = self.recenter(np.asarray(image.convert("RGBA")), border_ratio=border_ratio)
        else:
            raise TypeError("image must be a path or a PIL image")
        rgb = cv2.resize(rgb, (self.size, self.size), interpolation=cv2.INTER_CUBIC)
        mask = cv2.resize(mask, (self.size, self.size), interpolation=cv2.INTER_NEAREST)[..., None]
        if to_tensor:
            return array_to_tensor(rgb), array_to_tensor(mask)
        return rgb, mask

    def __call__(self, image, border_ratio=0.15, to_tensor=True, **kwargs):
        if self.border_ratio is not None:
            border_ratio = self.border_ratio
        img, mask = self.load_image(image, border_ratio=border_ratio, to_tensor=to_tensor)
        return {"image": img, "mask": mask}


class MVImageProcessorV2(ImageProcessorV2):
    """Multi-view input of Hunyuan3D-2mv (preprocessors.py:120-159): a dict {view tag: path or PIL image} with tags
    front (0), left (1), back (2), right (3), i.e. the front view turned clockwise by 0, 90, 180 and 270 degrees.  Each
    view goes through ImageProcessorV2; the views are ordered by index whatever the dict order, and stacked into
    image [1, V, 3, S, S], mask [1, V, 1, S, S] plus the sorted `view_idxs` tuple.  An unknown tag raises KeyError."""
    return_view_idx = True
    VIEW_INDEX = {"front": 0, "left": 1, "back": 2, "right": 3}

    def __init__(self, size=512, border_ratio=None):
        super().__init__(size, border_ratio)
        self.view2idx = dict(self.VIEW_INDEX)

    def __call__(self, image_dict, border_ratio=0.15, to_tensor=True, **kwargs):
        if self.border_ratio is not None:
            border_ratio = self.border_ratio
        views = []
        for tag, image in image_dict.items():
            idx = self.view2idx[tag]            # KeyError on an unknown tag, before any image is loaded
            views.append((idx, *self.load_image(image, border_ratio=border_ratio, to_tensor=to_tensor)))
        views.sort(key=lambda v: v[0])          # dict keys are distinct, so are their indices
        idxs, imgs, masks = zip(*views)
        return {"image": torch.cat(imgs, 0)[None], "mask": torch.cat(masks, 0)[None], "view_idxs": idxs}


IMAGE_PROCESSORS = {"v2": ImageProcessorV2, "mv_v2": MVImageProcessorV2}
DEFAULT_IMAGEPROCESSOR = "v2"
