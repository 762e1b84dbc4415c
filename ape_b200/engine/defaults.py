"""The predictor in front of the model (SURVEY.md §8(a) row 1, §8(f) row 3): `DefaultPredictor` of the reference
(ape/engine/defaults.py:159-230) with its input pipeline on the device.

Reference, per image and on the host: BGR -> RGB view (:218-220), `ResizeShortestEdge.get_transform(img).apply_image(img)`
(= PIL `Image.resize(BILINEAR)` for uint8 images, detectron2 `ResizeTransform.apply_image`), `astype("float32").transpose(2, 0, 1)`
(:221-222), the model's `.to(device)` of 12.6 MB of floats, then normalise + pad on the device.

Here: the raw uint8 HWC image goes through a pinned staging buffer to the device (3.1 MB at 1024^2, 0.8 MB for the 512^2 image
of BASELINE configs[0]), `ops.resize_u8_bilinear` reproduces Pillow's resample bit for bit (csrc/preprocess.cu) and writes
the float32 CHW tensor the input dict carries, with the channel flip folded into the write.  `predict_batch` overlaps the
upload + resize of image i+1 (side stream) with the forward of image i.

The mirrored names (`ResizeShortestEdge`, `DefaultPredictor.__call__(original_image, text_prompt, mask_prompt)`) take the
reference's arguments with the reference's meaning; what differs is stated in the docstrings."""
import sys

import numpy as np
import torch
import torch.nn.functional as F

from .. import ops


class ResizeTransform:
    """detectron2.data.transforms.ResizeTransform(h, w, new_h, new_w, interp=BILINEAR): `apply_image` on the device.
    uint8 images follow PIL (bit-exact, `ops.resize_u8_bilinear`); other dtypes follow detectron2's
    `F.interpolate(mode="bilinear", align_corners=False)` branch."""

    def __init__(self, h, w, new_h, new_w, interp=None):
        self.h, self.w, self.new_h, self.new_w = int(h), int(w), int(new_h), int(new_w)

    def apply_image(self, img, device="cuda", flip_channels=False, as_chw_float=True):
        """img: np.ndarray / torch tensor [H,W] or [H,W,C].  Returns a float32 device tensor [C,new_h,new_w] ([new_h,new_w]
        for 2-D input) — the tensor the reference's predictor builds on the host from apply_image's result."""
        t = torch.as_tensor(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
        assert tuple(t.shape[:2]) == (self.h, self.w), f"image of {tuple(t.shape[:2])} for a {self.h}x{self.w} transform"
        two_d = t.dim() == 2
        if t.dtype == torch.uint8:
            t = t.to(device, non_blocking=True)
            if not (t.stride(-1) == 1 and (two_d or t.stride(1) == t.shape[2])):
                t = t.contiguous()
            out = ops.resize_u8_bilinear(t, self.new_h, self.new_w, flip_channels=flip_channels and not two_d)
            return out[0] if two_d else out
        t = t.to(device, non_blocking=True).to(torch.float32)
        x = (t[None, None] if two_d else t.permute(2, 0, 1)[None])
        x = F.interpolate(x, (self.new_h, self.new_w), mode="bilinear", align_corners=False)[0]
        if flip_channels and not two_d:
            x = x.flip(0)
        return x[0] if two_d else x

    def apply_coords(self, coords):
        coords = np.asarray(coords, dtype=np.float64).copy()
        coords[:, 0] = coords[:, 0] * (self.new_w * 1.0 / self.w)
        coords[:, 1] = coords[:, 1] * (self.new_h * 1.0 / self.h)
        return coords


class NoOpTransform(ResizeTransform):
    def __init__(self, h, w):
        super().__init__(h, w, h, w)


class ResizeShortestEdge:
    """detectron2.data.transforms.ResizeShortestEdge(short_edge_length, max_size, sample_style): the test-time
    augmentation of every reference config (`configs/common/data/*_lsj1024.py`: short edge = max size = 1024)."""

    def __init__(self, short_edge_length, max_size=sys.maxsize, sample_style="range", interp=None):
        assert sample_style in ("range", "choice"), sample_style
        self.is_range = sample_style == "range"
        if isinstance(short_edge_length, int):
            short_edge_length = (short_edge_length, short_edge_length)
        if self.is_range:
            assert len(short_edge_length) == 2, f"short_edge_length must be two values using 'range' sample style. Got {short_edge_length}!"
        self.short_edge_length, self.max_size, self.sample_style = tuple(short_edge_length), max_size, sample_style

    def get_transform(self, image):
        h, w = image.shape[:2]
        if self.is_range:
            size = np.random.randint(self.short_edge_length[0], self.short_edge_length[1] + 1)
        else:
            size = np.random.choice(self.short_edge_length)
        if size == 0:
            return NoOpTransform(h, w)
        newh, neww = ResizeShortestEdge.get_output_shape(h, w, size, self.max_size)
        return ResizeTransform(h, w, newh, neww)

    @staticmethod
    def get_output_shape(oldh, oldw, short_edge_length, max_size):
        """Target size with the shorter side = short_edge_length and the longer side <= max_size (same float arithmetic and
        the same `int(x + 0.5)` rounding as detectron2)."""
        h, w = oldh, oldw
        size = short_edge_length * 1.0
        scale = size / min(h, w)
        if h < w:
            newh, neww = size, scale * w
        else:
            newh, neww = scale * h, size
        if max(newh, neww) > max_size:
            scale = max_size * 1.0 / max(newh, neww)
            newh = newh * scale
            neww = neww * scale
        neww = int(neww + 0.5)
        newh = int(newh + 0.5)
        return (newh, neww)


class DefaultPredictor:
    """`DefaultPredictor(cfg)` of the reference (ape/engine/defaults.py:159-230) for an already built engine model.

        pred = DefaultPredictor(model, aug=ResizeShortestEdge(1024, 1024), input_format="RGB")
        outputs = pred(cv2.imread("input.jpg"))                       # BGR uint8 HWC, as in the reference
        outputs = pred(img, text_prompt="person,traffic light")       # defaults.py:224-226
        outputs = pred(img, mask_prompt=mask)                         # defaults.py:227-229

    `from_cfg(cfg)` takes the reference's LazyConfig object (instantiate(cfg.model), checkpoint, test augmentation,
    input format: defaults.py:190-201) when detectron2 is importable.  Differences from the reference: the image is resized
    on the device (bit-exact with PIL for uint8 input) and `inputs["image"]` is a device tensor; the model is unchanged."""

    def __init__(self, model, aug=None, input_format="RGB"):
        assert input_format in ["RGB", "BGR"], input_format
        self.model = model.eval()
        self.aug = aug if aug is not None else ResizeShortestEdge(1024, 1024)
        self.input_format = input_format
        self.device = model.device if hasattr(model, "device") else next(model.parameters()).device
        self._staging = [None, None]  # pinned host buffers, alternated by predict_batch
        self._staged = [None, None]   # event after the last upload out of each buffer
        self._side = None

    @classmethod
    def from_cfg(cls, cfg):
        from detectron2.checkpoint import DetectionCheckpointer  # the reference's own dependencies: only needed on this route
        from detectron2.config import instantiate

        model = instantiate(cfg.model)
        model.to(cfg.train.device)
        DetectionCheckpointer(model).load(cfg.train.init_checkpoint)
        aug = cfg.dataloader.test.mapper.augmentations[0]
        aug = ResizeShortestEdge(aug.short_edge_length, aug.max_size, getattr(aug, "sample_style", "range"))
        fmt = cfg.model.model_vision.input_format if "model_vision" in cfg.model else cfg.model.input_format
        return cls(model, aug, fmt)

    # -- input pipeline ------------------------------------------------------------------------------------------
    def _upload(self, image, slot):
        """uint8 ndarray -> device tensor through a pinned staging buffer (reused per slot; the async copy is ordered on the
        current stream)."""
        if not (isinstance(image, np.ndarray) and image.dtype == np.uint8):
            return image
        n = int(image.size)
        ent = self._stage(slot, n)
        np.copyto(ent[1][:n].reshape(image.shape), image)  # one plain memcpy (a torch CPU copy_ spins up the intra-op pool)
        dev = ent[0][:n].view(image.shape).to(self.device, non_blocking=True)
        if self._staged[slot] is None:
            self._staged[slot] = torch.cuda.Event()
        self._staged[slot].record(torch.cuda.current_stream(self.device))
        return dev

    def _stage(self, slot, n):
        """The pinned staging buffer of `slot` with room for n bytes, once the previous upload out of it has finished."""
        ent = self._staging[slot]
        if ent is None or ent[0].numel() < n:
            buf = torch.empty((max(n, 1 << 22),), dtype=torch.uint8, pin_memory=True)
            ent = self._staging[slot] = (buf, buf.numpy())  # the numpy view shares the pinned pages
        if self._staged[slot] is not None:
            self._staged[slot].synchronize()  # the previous upload out of this buffer has finished
        return ent

    def _decode(self, source, slot):
        """A JPEG path or file bytes -> the device uint8 HWC image in the model's channel order (ape_b200.engine.read_image).
        The compressed bytes go through the slot's pinned staging buffer and the decode runs on a side stream: the host waits
        for the decode alone (to read its status), not for the forward already queued on the current stream, which then
        waits for the image."""
        from .read import decode, file_bytes

        data = file_bytes(source)
        main = torch.cuda.current_stream(self.device)
        if self._side is None:
            self._side = torch.cuda.Stream(self.device)
        ent = self._stage(slot, 3 * len(data) + (1 << 16))  # scan + decoder tables + restart offsets (4 bytes per 2-byte marker)
        done = torch.cuda.Event()
        with torch.cuda.stream(self._side):
            image, status, _ = decode(data, self.input_format, self.device, host=ent[0])
            if self._staged[slot] is None:
                self._staged[slot] = torch.cuda.Event()
            self._staged[slot].record(self._side)
            done.record(self._side)
            if status is not None:
                ops.jpeg_check(status)  # reads the status word on the side stream: waits for the decode only
        main.wait_event(done)
        image.record_stream(main)
        return image

    def preprocess(self, original_image, text_prompt=None, mask_prompt=None, slot=0):
        """defaults.py:216-229 up to the model call: the input dict, with `image` resized on the device.  original_image: the
        BGR uint8 array of the reference, or a JPEG file (path or bytes), decoded on the device as read_image(path, format)
        would on the host; height / width are then those of the EXIF-oriented image."""
        from .read import is_encoded

        if is_encoded(original_image):
            decoded = self._decode(original_image, slot)  # already in the model's channel order
            height, width = decoded.shape[:2]
            tfm = self.aug.get_transform(decoded)
            image = tfm.apply_image(decoded, device=self.device, flip_channels=False)
        else:
            height, width = original_image.shape[:2]
            tfm = self.aug.get_transform(original_image)
            image = tfm.apply_image(self._upload(original_image, slot), device=self.device, flip_channels=self.input_format == "RGB")
        inputs = {"image": image, "height": height, "width": width}
        if text_prompt is not None:
            inputs["prompt"] = "text"
            inputs["text_prompt"] = text_prompt
        if mask_prompt is not None:
            inputs["mask_prompt"] = self.aug.get_transform(mask_prompt).apply_image(mask_prompt, device=self.device)
        return inputs

    def __call__(self, original_image, text_prompt=None, mask_prompt=None):
        """original_image: np.ndarray (H, W, C) in BGR order, or a JPEG file as a path or bytes (decoded on the device,
        ape_b200.engine.read_image).  Returns the model's output dict for this one image."""
        with torch.no_grad():
            return self.model([self.preprocess(original_image, text_prompt, mask_prompt)])[0]

    def predict_batch(self, images, text_prompt=None):
        """One image after the other through the same model (batch 1 per step, the reference's evaluation setting), software
        pipelined: while the device runs the forward of image i, the host stages, uploads and resizes image i+1 and unpacks the
        detections of image i-1 — the device never waits for the host between images.  Boxes-only configurations go through
        `model.forward_packed` (results stay on the device until one small pinned copy); configurations with masks / semantic /
        panoptic outputs run one by one (their post-processing synchronises).  `images` may mix arrays and JPEG files (paths
        or bytes); the device decode of image i+1 runs on a side stream under the forward of image i.  Returns the list of
        output dicts."""
        from ..parallel import unpack_packed

        m = getattr(self.model, "model_vision", self.model)
        with_masks = getattr(m, "semantic_on", False) or getattr(m, "panoptic_on", False) or \
            (getattr(m, "instance_on", True) and getattr(m, "test_mask_on", False))
        if with_masks or not hasattr(m, "forward_packed"):
            return [self(im, text_prompt) for im in images]
        outs, pending = [], None  # pending = (device rows of the previous image, index)
        stream = torch.cuda.current_stream(self.device)
        with torch.no_grad():
            for i in range(len(images) + 1):
                inp = self.preprocess(images[i], text_prompt, slot=i & 1) if i < len(images) else None
                host, done = None, None
                if pending is not None:  # D2H of the previous image's rows BEFORE the next forward is enqueued
                    host = torch.empty(pending.shape, dtype=pending.dtype, pin_memory=True)
                    host.copy_(pending, non_blocking=True)
                    done = torch.cuda.Event()
                    done.record(stream)
                pending = m.forward_packed([inp]) if inp is not None else None
                if host is not None:
                    done.synchronize()
                    r = unpack_packed(host)[0]
                    if r.pop("num_candidates") > getattr(m, "static_inference_cap", 1 << 30) and not getattr(m, "_static_overflowed", False):
                        r = self(images[i - 1], text_prompt)  # the candidate list overflowed: take the host-synchronised route
                    outs.append(r)
        return outs
