"""GPU checks of the packed validation chains: every model input the YOLO-NAS COCO, YOLO-NAS-POSE and ResNet-50 validation batches
make is the bf16 rounding of the unmodified reference chain's float32 output, bit for bit (tests/golden/validation_chains.pt), over
mixed source shapes and a short last batch; and Trainer validation and test() give the same loss and metric values for a packed
loader as for the tuple loader of the same batches, eager and with cuda_graph on the train side."""
import copy
import hashlib
import os

import numpy as np
import pytest
import torch

import validation_cases as VC

pytestmark = pytest.mark.gpu
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _loader(ds, collate, batch_size=4, drop_last=False):
    return torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=False, num_workers=0, collate_fn=collate, pin_memory=True, drop_last=drop_last)


def _datasets():
    return VC.detection_dataset(), VC.pose_dataset(), VC.imagenet_dataset(pil=True)


@pytest.mark.parametrize("chain", [0, 1, 2])
def test_packed_inputs_match_the_reference_bit_for_bit(chain):
    golden = VC.golden()
    name = ("detection", "pose", "imagenet")[chain]
    ds, collate = _datasets()[chain], VC.collates()[chain]
    shas, sizes = [], []
    for batch in _loader(ds, collate):  # 4 + a short last batch
        images, _ = batch.to_model_input("cuda")
        assert images.dtype == torch.bfloat16 and images.is_contiguous(memory_format=torch.channels_last) and images.shape[1] == 16
        assert not images[:, 3:].any()
        sizes.append(images.shape[0])
        shas += [hashlib.sha256(x[:3].contiguous().view(torch.int16).cpu().numpy().tobytes()).hexdigest() for x in images]
    assert sizes[-1] < sizes[0]
    assert shas == [r["input_sha256"] for r in golden[name]["rows"]]


def _tiny_yolo_nas():
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    g = torch.load(os.path.join(HERE, "tiny_yolo_nas.pt"), weights_only=False)
    ap = copy.deepcopy(g["arch"])
    m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g["sd0"].items()}, strict=False)
    return m.cuda().train()


def _tiny_pose():
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPose

    g0 = torch.load(os.path.join(HERE, "tiny_yolo_nas_pose.pt"), weights_only=False)
    ap = copy.deepcopy(g0["arch"])
    m = YoloNASPose(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=5, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
    m.load_state_dict({k: v.clone() for k, v in g0["sd0"].items()}, strict=False)
    return m.cuda().train()


def _task(name):
    """(model, loss, metrics factory, packed batches list) of one task; the detection labels are folded onto the tiny model's 4
    classes and the pose stub has the tiny model's 5 joints."""
    from super_gradients_b200.training.datasets.detection_augment_dataset import CrowdDetectionAugmentCollateFN, DetectionAugmentDataset
    from super_gradients_b200.training.datasets.pose_estimation_datasets.pose_augment_dataset import PoseAugmentDataset, YoloNASPoseAugmentCollateFN
    from super_gradients_b200.training.losses import PPYoloELoss, YoloNASPoseLoss
    from super_gradients_b200.training.metrics import Accuracy, DetectionMetrics_050_095, PoseEstimationMetrics, Top5
    from super_gradients_b200.training.models import model_factory as models
    from super_gradients_b200.training.transforms import keypoints as KP
    from super_gradients_b200.training.transforms import transforms as T

    if name == "detection":
        stub = VC.StubDetectionDataset()
        for s in stub.samples:
            s["target"][:, 4] %= 4
            s["crowd_target"][:, 4] %= 4
        ds = DetectionAugmentDataset(stub, VC.build(VC.DETECTION, T), with_crowd=True)
        net = _tiny_yolo_nas()
        cb = net.get_post_prediction_callback(conf=0.01, iou=0.7, nms_top_k=1000, max_predictions=300, multi_label_per_box=True, class_agnostic_nms=False)
        return net, PPYoloELoss(num_classes=4, use_static_assigner=False), lambda: [DetectionMetrics_050_095(num_cls=4, post_prediction_callback=cb)], \
            _loader(ds, CrowdDetectionAugmentCollateFN.for_dataset(ds), 4)  # fmt: skip
    if name == "pose":
        g = torch.load(os.path.join(HERE, "tiny_yolo_nas_pose_train.pt"), weights_only=False)
        ds = PoseAugmentDataset(VC.StubValidationPoseDataset(num_joints=5), VC.build(VC.POSE, KP), with_gt_samples=True)
        net = _tiny_pose()
        cb = net.get_post_prediction_callback(conf=0.01, iou=0.7)
        return net, YoloNASPoseLoss(oks_sigmas=g["sigmas"], **g["kw"]), lambda: [PoseEstimationMetrics(post_prediction_callback=cb, num_joints=5, oks_sigmas=g["sigmas"])], \
            _loader(ds, YoloNASPoseAugmentCollateFN.for_dataset(ds), 4)  # fmt: skip
    ds = VC.imagenet_dataset(pil=True)
    return models.get("resnet18", num_classes=1000).cuda().train(), "CrossEntropyLoss", lambda: [Accuracy(), Top5()], _loader(ds, VC.collates()[2], 4)


def _tuple_batches(loader):
    """The tuple loader of the same batches: (model input, targets, extras) as the reference's collates give them, the input already
    the bf16 tensor the float batch becomes (checked bit for bit above)."""
    out = []
    for b in loader:
        images, targets = b.to_model_input("cuda")
        extras = getattr(b, "extras", {})
        out.append((images.clone(), targets, extras) if extras else (images.clone(), targets))
    return out


@pytest.mark.parametrize("cuda_graph", [False, True])
@pytest.mark.parametrize("name", ["detection", "pose", "classification"])
def test_trainer_validation_and_test_match_the_tuple_loader(tmp_path, name, cuda_graph):
    from super_gradients_b200.training.sg_trainer import Trainer

    torch.manual_seed(0)
    net, loss, metrics, packed = _task(name)
    tuples = _tuple_batches(packed)
    tp = dict(max_epochs=1, initial_lr=1e-3, lr_mode="constant", optimizer="SGD", loss=loss, cuda_graph=cuda_graph, save_model=False, valid_metrics_list=metrics(),
              silent_mode=True)  # fmt: skip
    tr = Trainer(f"val_{name}_{int(cuda_graph)}", ckpt_root_dir=str(tmp_path))
    train = _loader(packed.dataset, packed.collate_fn, 4, drop_last=True)  # one fixed-shape step for the captured graph
    tr.train(net, tp, train, valid_loader=packed)
    validated = {"valid_loss": tr.history["valid_loss"][-1], **tr.valid_metric_values}
    assert np.isfinite(validated["valid_loss"])
    results = []
    for loader in (packed, tuples):
        results.append(tr.test(test_loader=loader, test_metrics_list=metrics(), use_ema_net=False))
    assert results[0] == results[1]
    valid_loss, _, values = tr._evaluate(tuples, metrics())  # the validation train() ran, over the tuple loader
    assert {"valid_loss": valid_loss, **values} == validated
