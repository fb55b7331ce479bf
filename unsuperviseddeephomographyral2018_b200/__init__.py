"""H100-native unsupervised deep homography hot path (see DESIGN.md).

Public surface (mirrors the reference's names for this path):
    homography_model.HomographyModel, homography_model.homography_model_params
    ops.transformer, ops.solve_dlt, ops.warp_photo_loss
    dataloader.Dataloader, dataloader.dataloader_params
    engine.HomographyEngine (flat parameters, one-call steps, data parallelism), trainer.HostStepper (host-buffer API)
All arithmetic runs in libudh.so (include/udh.h); importing a submodule builds / loads it and fails loudly otherwise.
"""
__all__ = ["homography_model", "ops", "dataloader", "engine", "trainer", "synthetic", "params"]
