"""The GlobalConfig fields (team_code_transfuser/config.py:3-204) that the training hot path reads, with
train.py's CLI defaults applied (train.py:50-61: regnety_032 trunks, n_layer 4, use_velocity 0, use_target_point_image 1).
The reference's own `GlobalConfig` instance works unchanged with transfuser_b200.LidarCenterNet; this class exists so that
bench.py / smoke() / the GPU tests can run where no reference checkout exists."""


class TrainConfig:
    # data / geometry (config.py:5-31)
    seq_len = 1
    img_seq_len = 1
    lidar_seq_len = 1
    pred_len = 4
    lidar_resolution_width = 256
    lidar_resolution_height = 256
    lidar_pos = [1.3, 0.0, 2.5]
    bev_resolution_width = 160
    bev_resolution_height = 160
    use_target_point_image = True        # train.py:59
    gru_concat_target_point = True
    use_point_pillars = False
    max_lidar_points = 40000
    backbone = 'transFuser'
    # inference-side box decode (config.py:16, 39, 58-62)
    pixels_per_meter = 8.0
    bb_confidence_threshold = 0.3
    top_k_center_keypoints = 100
    center_net_max_pooling_kernel = 3
    bounding_box_divisor = 2.0
    # CenterNet (config.py:52-60)
    num_dir_bins = 12
    fp16_enabled = False
    channel = 64
    gru_hidden_size = 64
    num_class = 7
    # optimisation (config.py:119-123)
    lr = 1e-4
    multitask = True
    ls_seg = 1.0
    ls_depth = 10.0
    # encoders (config.py:126-147)
    img_vert_anchors = 5
    img_horz_anchors = 22
    lidar_vert_anchors = 8
    lidar_horz_anchors = 8
    detailed_losses = ['loss_wp', 'loss_bev', 'loss_depth', 'loss_semantic', 'loss_center_heatmap', 'loss_wh', 'loss_offset',
                       'loss_yaw_class', 'loss_yaw_res', 'loss_velocity', 'loss_brake']
    detailed_losses_weights = [1.0, 1.0, 1.0, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.0, 0.0]
    perception_output_features = 512
    bev_features_chanels = 64
    bev_upsample_factor = 2
    deconv_channel_num_1 = 128
    deconv_channel_num_2 = 64
    deconv_channel_num_3 = 32
    deconv_scale_factor_1 = 8
    deconv_scale_factor_2 = 4
    # GPT (config.py:174-185; n_layer 4 per train.py:56)
    n_embd = 512
    block_exp = 4
    n_layer = 4
    n_scale = 4
    n_head = 4
    embd_pdrop = 0.1
    resid_pdrop = 0.1
    attn_pdrop = 0.1
    gpt_linear_layer_init_mean = 0.0
    gpt_linear_layer_init_std = 0.02
    gpt_layer_norm_init_weight = 1.0
    # CARLA semantic tag -> the 7 training classes (config.py:88-117), used by the GPU input pipeline's class LUT
    converter = [0, 0, 0, 0, 4, 0, 5, 2, 6, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 3, 3, 0, 0, 5]

    def __init__(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self, k, v)
