"""CustomizableDetector: backbone -> neck -> heads from nested arch params
(reference: training/models/detection_models/customizable_detector.py:28-372)."""
from typing import Optional

import torch
from torch import nn

from .... import functional as SF
from ....common.factories import DetectionModulesFactory
from ..sg_module import SgModule


class CustomizableDetector(SgModule):
    def __init__(self, backbone, heads, neck=None, num_classes: int = None, bn_eps: Optional[float] = None, bn_momentum: Optional[float] = None, inplace_act: Optional[bool] = True, in_channels: int = 3):
        super().__init__()
        self.heads_params = heads
        self.bn_eps, self.bn_momentum, self.inplace_act, self.in_channels = bn_eps, bn_momentum, inplace_act, in_channels
        factory = DetectionModulesFactory()
        if num_classes is not None:
            self.heads_params = factory.insert_module_param(self.heads_params, "num_classes", num_classes)
        self.backbone = factory.get(factory.insert_module_param(backbone, "in_channels", in_channels))
        if neck is not None:
            self.neck = factory.get(factory.insert_module_param(neck, "in_channels", self.backbone.out_channels))
            self.heads = factory.get(factory.insert_module_param(heads, "in_channels", self.neck.out_channels))
        else:
            self.neck = nn.Identity()
            self.heads = factory.get(factory.insert_module_param(heads, "in_channels", self.backbone.out_channels))
        self._initialize_weights(bn_eps, bn_momentum, inplace_act)
        self._class_names = None
        self._image_processor = None
        self._default_nms_iou: float = 0.7
        self._default_nms_conf: float = 0.5
        self._default_nms_top_k: int = 1024
        self._default_max_predictions = 300
        self._default_multi_label_per_box = True
        self._default_class_agnostic_nms = False

    def forward(self, x):
        """x: [B, C, H, W] fp32 or bf16 CUDA tensor (NCHW semantics).  Same return structure as the reference."""
        stem = getattr(getattr(self.backbone, "stem", None), "conv", None)
        if stem is None or not hasattr(stem, "partially_fused") or not SF.stem_patches_supported(stem, x):
            x = SF.to_nhwc(x)  # else: the raw image goes to the stem, which gathers its patches itself (functional._QARepVGGStem)
        x = self.backbone(x)
        x = self.neck(x)
        return self.heads(x)

    def _initialize_weights(self, bn_eps=None, bn_momentum=None, inplace_act=True):
        for m in self.modules():
            if type(m) is nn.BatchNorm2d:
                m.eps = bn_eps if bn_eps else m.eps
                m.momentum = bn_momentum if bn_momentum else m.momentum

    def prep_model_for_conversion(self, input_size=None, **kwargs):
        for module in self.modules():
            if module != self and hasattr(module, "prep_model_for_conversion"):
                module.prep_model_for_conversion(input_size, **kwargs)

    def replace_head(self, new_num_classes: Optional[int] = None, new_head: Optional[nn.Module] = None):
        if new_num_classes is None and new_head is None:
            raise ValueError("At least one of new_num_classes, new_head must be given to replace output layer.")
        if new_head is not None:
            self.heads = new_head
        else:
            self.heads.replace_num_classes(new_num_classes, None)

    def replace_input_channels(self, in_channels: int, compute_new_weights_fn=None):
        """customizable_detector.py:124-129."""
        if not hasattr(self.backbone, "replace_input_channels"):
            raise NotImplementedError(f"`{self.backbone.__class__.__name__}` does not support `replace_input_channels`")
        self.backbone.replace_input_channels(in_channels=in_channels, compute_new_weights_fn=compute_new_weights_fn)
        self.in_channels = self.get_input_channels()

    def get_input_channels(self) -> int:
        return self.backbone.get_input_channels()

    def get_post_prediction_callback(self, *, conf: float, iou: float, nms_top_k: int, max_predictions: int, multi_label_per_box: bool, class_agnostic_nms: bool):
        raise NotImplementedError

    def set_dataset_processing_params(self, class_names=None, image_processor=None, iou=None, conf=None, nms_top_k=None, max_predictions=None, multi_label_per_box=None, class_agnostic_nms=None):
        if class_names is not None:
            self._class_names = tuple(class_names)
        if image_processor is not None:
            self._image_processor = image_processor
        if iou is not None:
            self._default_nms_iou = float(iou)
        if conf is not None:
            self._default_nms_conf = float(conf)
        if nms_top_k is not None:
            self._default_nms_top_k = int(nms_top_k)
        if max_predictions is not None:
            self._default_max_predictions = int(max_predictions)
        if multi_label_per_box is not None:
            self._default_multi_label_per_box = bool(multi_label_per_box)
        if class_agnostic_nms is not None:
            self._default_class_agnostic_nms = bool(class_agnostic_nms)

    def get_dataset_processing_params(self):
        """customizable_detector.py:197-207, including its `conf=self._default_nms_iou` (DESIGN.md section 4)."""
        return dict(class_names=self._class_names, image_processor=self._image_processor, iou=self._default_nms_iou, conf=self._default_nms_iou,
                    nms_top_k=self._default_nms_top_k, max_predictions=self._default_max_predictions, multi_label_per_box=self._default_multi_label_per_box,
                    class_agnostic_nms=self._default_class_agnostic_nms)  # fmt: skip

    def get_processing_params(self):
        return self._image_processor

    def image_processor_for_predict(self, skip_image_resizing: bool = False):
        """The chain predict() runs on raw images: the model's image processor -- the YOLO-NAS COCO chain when none was set, where the
        reference's pipeline raises (DESIGN.md section 4.9) -- or with skip_image_resizing its equivalent without resizing."""
        from ...processing import default_yolo_nas_coco_processing_params

        return (self._image_processor or default_yolo_nas_coco_processing_params()["image_processor"]).for_predict(skip_image_resizing)

    @torch.no_grad()
    def predict(self, images, iou=None, conf=None, batch_size: int = 32, fuse_model: bool = True, skip_image_resizing: bool = False, nms_top_k=None, max_predictions=None,
                multi_label_per_box=None, class_agnostic_nms=None, fp16: bool = True):  # fmt: skip
        """images: either a pre-processed tensor [B, C, H, W], or raw images -- one uint8 H x W x C array or a list of them (any
        sizes) -- which go through the model's image processor (set_dataset_processing_params; default: the YOLO-NAS COCO chain)
        as ONE fused GPU launch per image (training/processing/processing.py) and whose boxes come back in original-image pixels,
        like the reference's Pipeline (training/pipelines/pipelines.py:192-216).  skip_image_resizing: the chain without its resizing
        steps, padded bottom / right to a multiple of 32.  fp16 is accepted for the reference's signature: the model always runs its
        bf16 kernels.  Returns a list (one per image) of [Ni, 6] tensors (x1, y1, x2, y2, confidence, class)."""
        if not torch.is_tensor(images):
            return self._predict_raw_images(images, dict(iou=iou, conf=conf, nms_top_k=nms_top_k, max_predictions=max_predictions, multi_label_per_box=multi_label_per_box,
                                                         class_agnostic_nms=class_agnostic_nms), batch_size, skip_image_resizing)  # fmt: skip
        cb = self.get_post_prediction_callback(
            conf=self._default_nms_conf if conf is None else conf,
            iou=self._default_nms_iou if iou is None else iou,
            nms_top_k=self._default_nms_top_k if nms_top_k is None else nms_top_k,
            max_predictions=self._default_max_predictions if max_predictions is None else max_predictions,
            multi_label_per_box=self._default_multi_label_per_box if multi_label_per_box is None else multi_label_per_box,
            class_agnostic_nms=self._default_class_agnostic_nms if class_agnostic_nms is None else class_agnostic_nms,
        )
        was_training = self.training
        self.eval()
        out = []
        for i in range(0, images.shape[0], batch_size):
            out += cb(self(images[i : i + batch_size]))
        self.train(was_training)
        return out

    def _predict_raw_images(self, images, kw, batch_size, skip_image_resizing=False):
        import numpy as np

        images = [images] if isinstance(images, np.ndarray) else list(images)
        processor = self.image_processor_for_predict(skip_image_resizing)
        device = next(self.parameters()).device
        dflt = dict(conf=self._default_nms_conf, iou=self._default_nms_iou, nms_top_k=self._default_nms_top_k, max_predictions=self._default_max_predictions,
                    multi_label_per_box=self._default_multi_label_per_box, class_agnostic_nms=self._default_class_agnostic_nms)  # fmt: skip
        cb = self.get_post_prediction_callback(**{k: dflt[k] if kw.get(k) is None else kw[k] for k in dflt})
        was_training = self.training
        self.eval()
        out = []
        for i in range(0, len(images), batch_size):
            # one fused pre-processing launch per image, ONE model / decode / NMS pass per batch, padding / rescaling undone for the whole
            # batch at once, ONE device -> host copy; the per-image results are host views (the reference's pipeline returns host arrays)
            batch, geos = processor.preprocess_batch(images[i : i + batch_size], device)
            rows, _idx, count = cb.forward_batched(self(batch))
            shift, scale = processor.batch_shift_scale(geos, device)
            rows = torch.cat([(rows[..., :4] + shift.repeat(1, 2)[:, None, :]) * scale.repeat(1, 2)[:, None, :], rows[..., 4:]], dim=-1)
            rows_h, counts = rows.cpu(), count.tolist()
            out += [rows_h[b, :n] for b, n in enumerate(counts)]
        self.train(was_training)
        return out
