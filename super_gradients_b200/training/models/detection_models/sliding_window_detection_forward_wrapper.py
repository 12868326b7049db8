"""SlidingWindowInferenceDetectionWrapper (reference: training/models/detection_models/sliding_window_detection_forward_wrapper.py,
SG 3.7.1): detection on large images by running the model on overlapping square tiles and merging the tiles' detections with one
class-aware NMS per image.

The reference calls the model once per tile at batch 1, runs the post-prediction callback per tile, builds the per-image lists in
Python and calls torchvision's batched_nms once per image.  Here every predict batch (or forward() batch) costs: the pre-processing
launches, then per chunk of tiles one gather launch (csrc/sliding_window.cu), one model pass and one per-tile NMS launch (csrc/nms.cu)
writing into one buffer for the whole batch, then one merge (csrc/sliding_window.cu: compaction, sort, blocked greedy NMS per class)
and one device -> host copy.  No Python loop over tiles and no host synchronisation between chunks."""
from typing import List, Optional, Tuple

import numpy as np
import torch
from torch import nn

from .... import kernels as K
from .... import lib as L

# Tiles per model pass at 640 x 640 (the batch of bench config 5); smaller tiles take proportionally more.
_CHUNK_TILES_640 = 64


def tile_origins(height: int, width: int, tile_size: int, tile_step: int, min_tile_threshold: int) -> List[Tuple[int, int]]:
    """(y0, x0) of every tile of an image, y outer and x inner (_generate_tiles, :135-156).  A remainder below min_tile_threshold
    is not covered; otherwise the grid extends past the image, which reads as zeros.  The remainders use Python's modulo, also for
    an image smaller than a tile, which can leave it with no tile at all."""
    max_y = height if (height - tile_size) % tile_step < min_tile_threshold else height - (height - tile_size) % tile_step + tile_size
    max_x = width if (width - tile_size) % tile_step < min_tile_threshold else width - (width - tile_size) % tile_step + tile_size
    return [(y, x) for y in range(0, max_y - tile_size + 1, tile_step) for x in range(0, max_x - tile_size + 1, tile_step)]


def chunk_tiles(tile_size: int) -> int:
    """Tiles per model pass: a constant number of pixels, 64 tiles at 640 x 640."""
    return max(1, (_CHUNK_TILES_640 * 640 * 640) // (tile_size * tile_size))


class SlidingWindowInferenceDetectionWrapper(nn.Module):
    """Sliding-window inference for a CustomizableDetector (YOLO-NAS).

    :param tile_size:          side of the square tiles, in pixels of the model input.
    :param tile_step:          step between consecutive tiles.
    :param model:              the detector.
    :param min_tile_threshold: a remainder of the image narrower than this after the last full step gets no tile.
    :param tile_nms_*:         the per-tile post-prediction callback of forward(); unset values take the wrapper's defaults (iou 0.7,
                               conf 0.5, top-k 1024, 300 predictions per tile, multi-label, class-aware).  predict() builds its own
                               callback from its arguments and the same defaults (DESIGN.md section 4)."""

    def __init__(self, tile_size: int, tile_step: int, model, min_tile_threshold: int = 30, tile_nms_iou: Optional[float] = None, tile_nms_conf: Optional[float] = None,
                 tile_nms_top_k: Optional[int] = None, tile_nms_max_predictions: Optional[int] = None, tile_nms_multi_label_per_box: Optional[bool] = None,
                 tile_nms_class_agnostic_nms: Optional[bool] = None):  # fmt: skip
        super().__init__()
        self.tile_size = tile_size
        self.tile_step = tile_step
        self.min_tile_threshold = min_tile_threshold
        self._class_names = None
        self._image_processor = None
        self._default_nms_iou: float = 0.7
        self._default_nms_conf: float = 0.5
        self._default_nms_top_k: int = 1024
        self._default_max_predictions = 300
        self._default_multi_label_per_box = True
        self._default_class_agnostic_nms = False
        self.model = model
        # :68-95: the model's processing parameters (class names, image processor) first; the tile callback then comes from the
        # explicit tile_nms_* over the wrapper's defaults -- never from the model's NMS defaults
        self.set_dataset_processing_params(**self.model.get_dataset_processing_params())
        self.set_dataset_processing_params(iou=tile_nms_iou, conf=tile_nms_conf, nms_top_k=tile_nms_top_k, max_predictions=tile_nms_max_predictions,
                                           multi_label_per_box=tile_nms_multi_label_per_box, class_agnostic_nms=tile_nms_class_agnostic_nms)  # fmt: skip

    def get_post_prediction_callback(self, *, conf: float, iou: float, nms_top_k: int, max_predictions: int, multi_label_per_box: bool, class_agnostic_nms: bool):
        return self.model.get_post_prediction_callback(conf=conf, iou=iou, nms_top_k=nms_top_k, max_predictions=max_predictions, multi_label_per_box=multi_label_per_box,
                                                       class_agnostic_nms=class_agnostic_nms)  # fmt: skip

    def set_dataset_processing_params(self, class_names=None, image_processor=None, iou=None, conf=None, nms_top_k=None, max_predictions=None, multi_label_per_box=None,
                                      class_agnostic_nms=None) -> None:  # fmt: skip
        """:179-230: class names and image processor are stored; the NMS values rebuild forward()'s tile callback over the wrapper's
        defaults, which they do not change."""
        if class_names is not None:
            self._class_names = tuple(class_names)
        if image_processor is not None:
            self._image_processor = image_processor
        self.sliding_window_post_prediction_callback = self._callback(iou, conf, nms_top_k, max_predictions, multi_label_per_box, class_agnostic_nms)

    def _callback(self, iou, conf, nms_top_k, max_predictions, multi_label_per_box, class_agnostic_nms):
        pick = lambda v, d: d if v is None else v  # noqa: E731
        return self.get_post_prediction_callback(iou=float(pick(iou, self._default_nms_iou)), conf=float(pick(conf, self._default_nms_conf)),
                                                 nms_top_k=int(pick(nms_top_k, self._default_nms_top_k)), max_predictions=int(pick(max_predictions, self._default_max_predictions)),
                                                 multi_label_per_box=bool(pick(multi_label_per_box, self._default_multi_label_per_box)),
                                                 class_agnostic_nms=bool(pick(class_agnostic_nms, self._default_class_agnostic_nms)))  # fmt: skip

    def get_processing_params(self):
        return self._image_processor

    def get_input_channels(self) -> int:
        return self.model.get_input_channels()

    @torch.no_grad()
    def forward(self, inputs: torch.Tensor, sliding_window_post_prediction_callback=None) -> List[torch.Tensor]:
        """inputs: [B, C, H, W] fp32 NCHW (converted on the device) or a bf16 NHWC canvas with 16 channels.  Returns the per-image
        list of [Ni, 6] rows (x1, y1, x2, y2, confidence, class) in input pixels, on the device."""
        cb = sliding_window_post_prediction_callback or self.sliding_window_post_prediction_callback
        canvas = inputs if inputs.dtype == torch.bfloat16 else K.nchw_f32_to_nhwc_bf16(inputs, 16)
        rows, count = self._detect(canvas, cb)
        counts = count.tolist()
        if min(counts, default=0) < 0:
            raise L.SgbError(f"sliding-window merge refused a malformed per-tile row (counts {counts})")
        return [rows[b, : counts[b]] for b in range(len(counts))]

    def _detect(self, canvas: torch.Tensor, cb) -> Tuple[torch.Tensor, torch.Tensor]:
        """canvas: bf16 NHWC [B, 16, H, W] -> (rows [B, cap, 6] in canvas pixels, count [B] int32), both on the device."""
        B, _, H, W = canvas.shape
        device = canvas.device
        origins = tile_origins(H, W, self.tile_size, self.tile_step, self.min_tile_threshold)
        if not origins:  # :127-130: an image without tiles has no detections
            return torch.zeros((B, 0, 6), dtype=torch.float32, device=device), torch.zeros((B,), dtype=torch.int32, device=device)
        per = len(origins)
        T = B * per
        on_gpu = device.type == "cuda"
        tiles_host = torch.tensor([(b, y, x) for b in range(B) for (y, x) in origins], dtype=torch.int32)
        image_tiles_host = torch.arange(0, T + 1, per, dtype=torch.int32)
        if on_gpu:
            tiles_host, image_tiles_host = tiles_host.pin_memory(), image_tiles_host.pin_memory()
        tiles = tiles_host.to(device, non_blocking=True)
        image_tiles = image_tiles_host.to(device, non_blocking=True)
        P = cb.max_rows()
        rows = torch.empty((T, P, 6), dtype=torch.float32, device=device)
        idx = torch.empty((T, P), dtype=torch.int32, device=device)
        count = torch.empty((T,), dtype=torch.int32, device=device)
        step = chunk_tiles(self.tile_size)
        ncls = None
        for c0 in range(0, T, step):
            c1 = min(T, c0 + step)
            batch = K.sliding_window_gather(canvas, tiles_host[c0:c1], tiles[c0:c1], self.tile_size)
            out = self.model(batch)
            ncls = cb._get_decoded_predictions_from_model_output(out)[1].shape[-1]
            cb.forward_batched(out, out=rows[c0:c1], out_idx=idx[c0:c1], out_count=count[c0:c1])
        return K.sliding_window_merge(rows, count, tiles, image_tiles_host, image_tiles, ncls, cb.nms_threshold)

    @torch.no_grad()
    def predict(self, images, iou: Optional[float] = None, conf: Optional[float] = None, batch_size: int = 32, fuse_model: bool = True, skip_image_resizing: bool = False,
                nms_top_k: Optional[int] = None, max_predictions: Optional[int] = None, multi_label_per_box: Optional[bool] = None, class_agnostic_nms: Optional[bool] = None,
                fp16: bool = True) -> List[torch.Tensor]:  # fmt: skip
        """images: one uint8 H x W x C array or a list of them; the images of one batch must map to one canvas.  Without an image
        processor (set_dataset_processing_params or the model's) the YOLO-NAS COCO chain runs, where the reference raises.  The tile callback is
        built from these arguments over the wrapper's defaults (_get_pipeline, :232-290), not from the constructor's tile_nms_*.
        skip_image_resizing: the chain without its resizing steps, padded bottom / right to a multiple of 32.  fuse_model and fp16
        are accepted for the reference's signature (the model always runs its bf16 kernels).  Returns a list (one per image) of
        [Ni, 6] host tensors (x1, y1, x2, y2, confidence, class) in original-image pixels."""
        from ...processing import default_yolo_nas_coco_processing_params

        images = [images] if isinstance(images, np.ndarray) else list(images)
        processor = (self._image_processor or default_yolo_nas_coco_processing_params()["image_processor"]).for_predict(skip_image_resizing)
        cb = self._callback(iou, conf, nms_top_k, max_predictions, multi_label_per_box, class_agnostic_nms)
        device = next(self.model.parameters()).device
        was_training = self.model.training
        self.model.eval()
        out = []
        try:
            for i in range(0, len(images), batch_size):
                canvas, geos = processor.preprocess_batch(images[i : i + batch_size], device)
                rows, count = self._detect(canvas, cb)
                shift, scale = processor.batch_shift_scale(geos, device)
                rows = torch.cat([(rows[..., :4] + shift.repeat(1, 2)[:, None, :]) * scale.repeat(1, 2)[:, None, :], rows[..., 4:]], dim=-1)
                # ONE device -> host copy: the rows with the counts' bits behind them
                host = torch.cat([rows.reshape(-1), count.view(torch.float32)]).cpu()
                nb = count.shape[0]
                counts = host[host.numel() - nb :].view(torch.int32).tolist()
                if min(counts) < 0:
                    raise L.SgbError(f"sliding-window merge refused a malformed per-tile row (counts {counts})")
                rows_h = host[: host.numel() - nb].view(rows.shape)
                out += [rows_h[b, :n] for b, n in enumerate(counts)]
        finally:
            self.model.train(was_training)
        return out
