"""Worker of tests/test_optimizers_cpu.py::test_trainer_world2_gloo: Trainer.train() of the tiny YOLO-NAS with Adam, RMSprop,
RMSpropTF, Lion and Lamb on every rank of a gloo group (CPU stand-in backend), each rank on its own shard; after every run the
ranks' flat parameters and optimizer states must be identical."""
import copy
import os
import subprocess
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main(ckpt_dir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    from _pytest.monkeypatch import MonkeyPatch

    import cpu_backend
    import host_optim

    from super_gradients_b200.training import sg_trainer
    from super_gradients_b200.training.losses import PPYoloELoss
    from super_gradients_b200.training.models.detection_models.yolo_nas import YoloNAS

    dist.init_process_group("gloo", init_method="env://")
    mp = MonkeyPatch()
    cpu_backend.install_training(mp)
    host_optim.install(mp)
    sg_trainer.setup_device = lambda device=None: torch.device("cpu")
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "tiny_yolo_nas.pt"), weights_only=False)
    rank = dist.get_rank()
    try:
        for name, params in (("Adam", {}), ("RMSprop", {"centered": True}), ("RMSpropTF", {}), ("Lion", {"weight_decay": 0.1}), ("Lamb", {"weight_decay": 0.01})):
            torch.manual_seed(0)
            ap = copy.deepcopy(fx["arch"])
            m = YoloNAS(backbone=ap["backbone"], neck=ap["neck"], heads=ap["heads"], num_classes=4, bn_eps=1e-3, bn_momentum=0.03, inplace_act=True, in_channels=3)
            m.load_state_dict({k: v.clone() for k, v in fx["sd0"].items()}, strict=False)
            tp = dict(max_epochs=1, initial_lr=1e-3, lr_mode="constant", optimizer=name, optimizer_params=params, zero_weight_decay_on_bias_and_bn=True,
                      loss=PPYoloELoss(num_classes=4, use_static_assigner=False), save_model=False)  # fmt: skip
            tr = sg_trainer.Trainer(name, ckpt_root_dir=ckpt_dir)
            hist = tr.train(m, tp, [(fx["x"] * (1.0 if rank == 0 else 0.9), fx["targets"])] * 2)
            assert all(torch.isfinite(torch.tensor(hist["train_loss"]))), name
            assert tr.step.world == 2
            for t in (tr.step.flat.params, *tr.step.state):
                both = [torch.zeros_like(t) for _ in range(2)]
                dist.all_gather(both, t)
                assert torch.equal(both[0], both[1]), f"{name}: replicas diverged"
        print("rank", rank, "optimizers ok", flush=True)
        dist.barrier()
    finally:
        mp.undo()
        dist.destroy_process_group()


def launch(ckpt_dir, port, timeout=900):
    """Runs main() on two ranks as direct child processes; -> (returncodes, combined output).  Every child is joined, or killed
    and reaped on timeout."""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE="2", OMP_NUM_THREADS="2")
    procs = []
    try:
        for r in range(2):
            procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), ckpt_dir], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT, text=True))  # fmt: skip
        deadline = time.monotonic() + timeout
        outs = [p.communicate(timeout=max(1.0, deadline - time.monotonic()))[0] for p in procs]
        return [p.returncode for p in procs], "\n".join(outs)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()


if __name__ == "__main__":
    main(sys.argv[1])
