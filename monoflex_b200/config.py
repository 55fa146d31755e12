"""The subset of the reference configuration the hot path reads (config/defaults.py + runs/monoflex.yaml), as a plain
attribute tree. Any object with the same attributes works (e.g. the reference's yacs CfgNode), so
`KeypointDetector(cfg)` accepts the reference's own `cfg` unchanged."""
from types import SimpleNamespace as NS


def default_cfg(width=1280, height=384, device="cuda"):
    cfg = NS()
    cfg.MODEL = NS(DEVICE=device, PRETRAIN=False, INPLACE_ABN=True, USE_SYNC_BN=False)
    cfg.MODEL.BACKBONE = NS(CONV_BODY="dla34", DOWN_RATIO=4)
    cfg.MODEL.HEAD = NS(
        PREDICTOR="Base_Predictor", NUM_CHANNEL=256, USE_NORMALIZATION="BN", BN_MOMENTUM=0.1, INIT_P=0.01,
        UNCERTAINTY_INIT=True,
        REGRESSION_HEADS=[['2d_dim'], ['3d_offset'], ['corner_offset'], ['corner_uncertainty'], ['3d_dim'],
                          ['ori_cls', 'ori_offset'], ['depth'], ['depth_uncertainty']],
        REGRESSION_CHANNELS=[[4], [2], [20], [3], [3], [8, 8], [1], [1]],
        ENABLE_EDGE_FUSION=True, EDGE_FUSION_KERNEL_SIZE=3, EDGE_FUSION_NORM='BN', EDGE_FUSION_RELU=False,
        DEPTH_MODE='inv_sigmoid', DEPTH_RANGE=[0.1, 100], OUTPUT_DEPTH='soft',
        DIMENSION_MEAN=((3.8840, 1.5261, 1.6286), (0.8423, 1.7607, 0.6602), (1.7635, 1.7372, 0.5968)),
        DIMENSION_REG=['exp', True, False],
        # training losses (runs/monoflex.yaml:34-47 over config/defaults.py:137-197)
        LOSS_TYPE=["Penalty_Reduced_FocalLoss", "L1", "giou", "L1"], HEATMAP_TYPE='centernet', LOSS_PENALTY_ALPHA=2, LOSS_BETA=4,
        LOSS_NAMES=['hm_loss', 'bbox_loss', 'depth_loss', 'offset_loss', 'orien_loss', 'dims_loss', 'corner_loss',
                    'keypoint_loss', 'keypoint_depth_loss', 'trunc_offset_loss', 'weighted_avg_depth_loss'],
        INIT_LOSS_WEIGHT=[1, 1, 1, 0.5, 1, 1, 0.2, 1.0, 0.2, 0.1, 0.2], CORNER_LOSS_DEPTH='soft_combine',
        TRUNCATION_OFFSET_LOSS='log', MODIFY_INVALID_KEYPOINT_DEPTH=True, UNCERTAINTY_RANGE=[-10, 10],
        DIMENSION_WEIGHT=[1, 1, 1])
    cfg.INPUT = NS(WIDTH_TRAIN=width, HEIGHT_TRAIN=height, WIDTH_TEST=width, HEIGHT_TEST=height,
                   ORIENTATION='multi-bin', ORIENTATION_BIN_SIZE=4)
    cfg.DATASETS = NS(DETECT_CLASSES=("Car", "Pedestrian", "Cyclist"), TEST_SPLIT="test", MAX_OBJECTS=40)
    cfg.TEST = NS(DETECTIONS_THRESHOLD=0.2, DETECTIONS_PER_IMG=50, UNCERTAINTY_AS_CONFIDENCE=True, PRED_2D=True,
                  EVAL_DIS_IOUS=False, EVAL_DEPTH=False)
    # runs/monoflex.yaml:61-78 over config/defaults.py:252-299
    cfg.SOLVER = NS(OPTIMIZER="adamw", BASE_LR=3e-4, WEIGHT_DECAY=1e-5, BIAS_LR_FACTOR=2.0, STEPS=(20000, 25000),
                    LR_DECAY=0.1, LR_CLIP=1e-7, LR_WARMUP=False, WARMUP_STEPS=2000, GRAD_NORM_CLIP=-1, IMS_PER_BATCH=8,
                    MAX_ITERATION=30000, MOMS=[0.95, 0.85], PCT_START=0.4, DIV_FACTOR=10)
    return cfg
