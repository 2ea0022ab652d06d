"""ctypes binding of libpcb200.so (include/pcb200.h).  There is NO fallback: if the library is missing or a call
fails, this raises."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "libpcb200.so")


class PcbError(RuntimeError):
    pass


def _load():
    if not os.path.exists(_PATH):
        raise ImportError(
            f"{_PATH} not found: the CUDA extension is not built. Run `python -m pointcontrast_b200.build` "
            "(needs nvcc; there is no CPU fallback).")
    return C.CDLL(_PATH)


lib = _load()

_p, _i, _l, _f, _d, _sz = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double, C.c_size_t

class PcbStrided(C.Structure):
    """`struct pcb_strided` of include/pcb200.h: a float tensor read through its element strides (scene, proposal, channel, xyz)."""
    _fields_ = [("p", _p), ("sb", _l), ("sk", _l), ("sc", _l), ("sx", _l)]


class PcbDetLossArgs(C.Structure):
    """`struct pcb_det_loss_args` of include/pcb200.h (field for field)."""
    _fields_ = [
        ("B", _l), ("S", _l), ("V", _l), ("N", _l), ("K", _l), ("K2", _l),
        ("NH", C.c_int32), ("NS", C.c_int32), ("C", C.c_int32), ("seed_inds_i64", C.c_int32),
        ("heading_scale", _f),
        ("mean_size", _p),
        ("seed_xyz", _p), ("seed_inds", _p), ("vote_xyz", _p), ("vote_label", _p), ("vote_label_mask", _p),
        ("aggregated_vote_xyz", _p),
        ("center", PcbStrided), ("objectness_scores", PcbStrided), ("heading_scores", PcbStrided),
        ("heading_residuals_normalized", PcbStrided), ("size_scores", PcbStrided), ("size_residuals_normalized", PcbStrided),
        ("sem_cls_scores", PcbStrided),
        ("center_label", _p), ("center_label_ld", _l),
        ("heading_class_label", _p), ("heading_residual_label", _p), ("size_class_label", _p),
        ("size_residual_label", _p), ("sem_cls_label", _p), ("box_label_mask", _p),
    ]


class PcbDetBatch(C.Structure):
    """`struct pcb_det_batch` of include/pcb200.h (field for field)."""
    _fields_ = [
        ("B", _l), ("M", _l), ("num_points", _l), ("dataset", C.c_int32), ("flags", C.c_int32),
        ("offsets_host", _p), ("offsets", _p), ("box_offsets_host", _p), ("box_offsets", _p),
        ("params", _p), ("floor", _p), ("choices", _p),
        ("vert", _p), ("sem", _p), ("ins", _p), ("pc", _p), ("votes", _p), ("jitter", _p), ("dropout", _p),
        ("boxes", _p), ("headings", _p), ("nyu40ids", _p), ("n_ids", C.c_int32), ("num_heading_bin", C.c_int32),
        ("mean_size", _p), ("n_size", C.c_int32), ("pad_", C.c_int32),
        ("point_clouds", _p), ("pcl_color", _p), ("vote_label", _p), ("vote_label_mask", _p),
        ("center_label", _p), ("heading_class_label", _p), ("heading_residual_label", _p), ("size_class_label", _p),
        ("size_residual_label", _p), ("sem_cls_label", _p), ("box_label_mask", _p), ("max_gt_bboxes", _p),
    ]


_DLA = C.POINTER(PcbDetLossArgs)
_DDB = C.POINTER(PcbDetBatch)
_PS = C.POINTER(PcbStrided)
_SIGS = {
    "pcb_last_error": (C.c_char_p, []),
    "pcb_version": (C.c_char_p, []),
    "pcb_launch_count": (C.c_uint64, []),
    "pcb_set_device": (_i, [_i]),
    "pcb_coords_pack": (_i, [_p, _l, _p, _p, _p]),
    "pcb_coords_unpack": (_i, [_p, _l, _p, _p]),
    "pcb_hash_build": (_i, [_p, _l, _p, _p, _l, _p, _p]),
    "pcb_coords_stride_ws_bytes": (_sz, [_l]),
    "pcb_coords_stride": (_i, [_p, _l, C.c_int32, _p, _p, C.POINTER(C.c_int64), _p, _sz, _p]),
    "pcb_voxelize_ws_bytes": (_sz, [_l]),
    "pcb_voxelize": (_i, [_p, _l, _f, _p, _p, C.POINTER(C.c_int64), _p, _sz, _p]),
    "pcb_radius_pairs_ws_bytes": (_sz, [_l, _l]),
    "pcb_radius_pairs": (_i, [_p, _l, _p, _l, _f, _p, _l, C.POINTER(C.c_int64), _p, _sz, _p]),
    "pcb_voxelize_labels_ws_bytes": (_sz, [_l]),
    "pcb_voxelize_labels": (_i, [_p, _p, _l, C.c_int32, _p, _p, _p, C.POINTER(C.c_int64), _p, _sz, _p]),
    "pcb_point_bounds_ws_bytes": (_sz, []),
    "pcb_point_bounds": (_i, [_p, _l, _p, _p, _p, _sz, _p]),
    "pcb_elastic_distort_ws_bytes": (_sz, [_i, _i, _i]),
    "pcb_elastic_distort": (_i, [_p, _l, _p, _i, _i, _i, _p, _d, _p, _sz, _p]),
    "pcb_affine_floor_ws_bytes": (_sz, []),
    "pcb_affine_floor": (_i, [_p, _l, _p, _p, _p, _p, _sz, _p]),
    "pcb_semseg_input_transform_ws_bytes": (_sz, []),
    "pcb_semseg_input_transform": (_i, [_p, _p, _l, _i, _i, _d, _p, _p, _d, _i, _p, _sz, _p]),
    "pcb_kernel_map": (_i, [_p, _l, _p, _p, _l, _p, _i, _p, _p]),
    "pcb_kernel_map_count": (_i, [_p, _i, _l, _p, _p]),
    "pcb_conv_tile_order_ws_bytes": (_sz, [_l]),
    "pcb_conv_tile_order": (_i, [_p, _l, _i, _l, _l, _p, _p, _sz, _p]),
    "pcb_conv_forward": (_i, [_p, _i, _p, _l, _p, _i, _l, _i, _i, _p, _p, _p, _i, _p]),
    "pcb_gather_sum": (_i, [_p, _i, _p, _l, _p, _i, _l, _i, _p, _i, _p, _p]),
    "pcb_conv_wgrad_ws_bytes": (_sz, [_i, _l, _i, _i]),
    "pcb_conv_wgrad": (_i, [_p, _i, _p, _i, _p, _l, _i, _l, _i, _i, _p, _i, _p, _sz, _i, _p]),
    "pcb_weight_tile_bytes": (_sz, [_i, _i, _i, _i]),
    "pcb_weight_tile": (_i, [_p, _i, _i, _i, _p, _p, _i, _p]),
    "pcb_tile_desc_fill": (_i, [_p, _p, _i, _i, _i, _p, _p, _i, _l]),
    "pcb_weight_tile_batch": (_i, [_p, _i, _l, _p]),
    "pcb_conv_forward_split_ws_bytes": (_sz, [_i, _l, _i, _i]),
    "pcb_conv_forward_split": (_i, [_p, _p, _i, _p, _l, _p, _i, _l, _i, _i, _p, _p, _p, _i, _p, _sz, _i, _p]),
    "pcb_conv_forward_split_ordered": (_i, [_p, _p, _i, _p, _l, _p, _i, _p, _l, _i, _i, _p, _p, _p, _i, _p, _sz, _i, _p]),
    "pcb_conv_wgrad_split_ws_bytes": (_sz, [_i, _l, _i, _i]),
    "pcb_conv_wgrad_split": (_i, [_p, _p, _i, _p, _p, _i, _p, _l, _i, _l, _i, _i, _p, _i, _p, _sz, _i, _p]),
    "pcb_bn_ws_bytes": (_sz, [_l, _i]),
    "pcb_bn_stats_seg": (_i, [_p, _i, _l, _l, _i, _f, _f, _p, _p, _p, _p, _p, _sz, _p]),
    "pcb_bn_apply_seg": (_i, [_p, _i, _l, _l, _i, _p, _p, _p, _p, _p, _i, _i, _p, _i, _p, _p, _i, _p, _p, _p]),
    "pcb_bn_backward_seg": (_i, [_p, _i, _p, _i, _p, _i, _l, _l, _i, _p, _p, _p, _p, _i, _p, _p, _i, _p, _i, _i, _p, _p, _i, _p, _sz,
                                 _p]),
    "pcb_split_rows": (_i, [_p, _i, _l, _i, _p, _p, _i, _i, _p]),
    "pcb_nce_ws_bytes": (_sz, [_l]),
    "pcb_nce_forward_backward": (_i, [_p, _p, _l, _i, _f, _p, _p, _p, _p, _sz, _p]),
    "pcb_l2norm_forward": (_i, [_p, _l, _i, _p, _p, _p]),
    "pcb_l2norm_backward": (_i, [_p, _p, _p, _l, _i, _p, _p]),
    "pcb_pdist_rowmin": (_i, [_p, _l, _p, _l, _i, _p, _p, _p, _p]),
    "pcb_sgd_step": (_i, [_p, _p, _p, _l, _f, _f, _f, _f, _i, _f, _p]),
    "pcb_ce_ws_bytes": (_sz, [_l]),
    "pcb_ce_forward_backward": (_i, [_p, _p, _l, _i, _l, _f, _p, _p, _p, _sz, _p]),
    "pcb_seg_metrics_ws_bytes": (_sz, [_l]),
    "pcb_seg_metrics": (_i, [_p, _p, _l, _i, _l, _p, _p, _p, _p, _p, _sz, _p]),
    "pcb_average_precision_ws_bytes": (_sz, [_l, _i]),
    "pcb_average_precision": (_i, [_p, _p, _l, _i, _p, _p, _p, _sz, _p]),
    "pcb_det_decode_pred": (_i, [_p, _p, _p, _p, _p, _p, _p, _l, _l, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _p]),
    "pcb_det_decode_gt": (_i, [_p, _p, _p, _p, _p, _l, _l, _i, _i, _p, _i, _p, _p, _p, _p]),
    "pcb_det_points_in_box": (_i, [_p, _l, _l, _i, _p, _l, _p, _p]),
    "pcb_det_nms": (_i, [_p, _p, _p, _p, _i, _l, _l, _i, _i, _d, _p, _p]),
    "pcb_det_box_iou": (_i, [_p, _p, _l, _p, _p]),
    "pcb_det_ap_ws_bytes": (_sz, [_l, _l, _i, _i]),
    "pcb_det_ap": (_i, [_p, _l, _p, _p, _p, _p, _l, _p, _p, _p, _l, _i, _p, _i, _p, _p, _sz, _p]),
    "pcb_det_loss_ws_bytes": (_sz, [_l, _l, _l, _l]),
    "pcb_det_loss_state_bytes": (_sz, [_l, _l, _l, _l]),
    "pcb_det_loss_forward": (_i, [_DLA, _p, _p, _p, _p, _p, _sz, _p, _sz, _p]),
    "pcb_det_loss_backward": (_i, [_DLA, _p, _p, _p, _p, _p, _sz, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "pcb_det_floor_height": (_i, [_p, _l, C.c_int32, _p, _p, _l, _p, _p]),
    "pcb_det_choices_ws_bytes": (_sz, [_l]),
    "pcb_det_choices": (_i, [_p, _p, _l, _l, C.c_uint64, C.c_uint64, _p, _p, _sz, _p]),
    "pcb_det_points_ws_bytes": (_sz, [_l, _l]),
    "pcb_det_points": (_i, [_DDB, _p, _sz, _p]),
    "pcb_det_boxes": (_i, [_DDB, _p]),
    "pcb_profile_enable": (_i, [_i]),
    "pcb_profile_read": (_i, [_p, _p, _i, C.POINTER(C.c_int)]),
    "pcb_unit_ws_bytes": (_sz, [_i, _l, _l, _i, _i]),
    "pcb_unit_forward": (_i, [_p, _p]),
    "pcb_unit_backward": (_i, [_p, _p]),
    "pcb_furthest_point_sampling_ws_bytes": (_sz, [_l, _l]),
    "pcb_furthest_point_sampling": (_i, [_p, _l, _l, _l, _p, _p, _sz, _p]),
    "pcb_ball_query": (_i, [_p, _p, _l, _l, _l, _f, _i, _p, _p]),
    "pcb_three_nn": (_i, [_p, _p, _l, _l, _l, _p, _p, _p]),
    "pcb_gather_points": (_i, [_p, _p, _l, _l, _l, _l, _p, _p]),
    "pcb_three_interpolate": (_i, [_p, _p, _p, _l, _l, _l, _l, _p, _p]),
    "pcb_points_grad_ws_bytes": (_sz, [_l, _l, _l]),
    "pcb_gather_points_grad": (_i, [_p, _p, _l, _l, _l, _l, _p, _p, _sz, _p]),
    "pcb_three_interpolate_grad": (_i, [_p, _p, _p, _l, _l, _l, _l, _p, _p, _sz, _p]),
    "pcb_voxelize_scenes_ws_bytes": (_sz, [_l, _l]),
    "pcb_voxelize_scenes": (_i, [_p, _l, _l, _f, _p, _p, _p, _p, _p, _sz, _p]),
    "pcb_furthest_point_sampling_ragged_ws_bytes": (_sz, [_l, _l, _l]),
    "pcb_furthest_point_sampling_ragged": (_i, [_p, _p, _l, _l, _l, _l, _p, _p, _sz, _p]),
    "pcb_gather_rows_grad": (_i, [_p, _p, _l, _l, _l, _p, _p, _sz, _p]),
    "pcb_sa_layer0": (_i, [_p, _p, _p, _l, _l, _l, _i, _f, _p, _i, _p, _i, _p, _p, _p, _i, _p]),
    "pcb_sa_pool": (_i, [_p, _i, _l, _i, _i, _p, _p, _p, _p, _p, _p, _i, _p]),
    "pcb_sa_pool_grad": (_i, [_p, _i, _p, _p, _i, _l, _i, _i, _p, _p]),
    "pcb_sa_xyz_rows": (_i, [_p, _p, _l, _i, _f, _p, _p]),
    "pcb_vote_epilogue": (_i, [_p, _p, _i, _p, _i, _l, _l, _i, _i, _p, _p, _p]),
    "pcb_vote_epilogue_grad": (_i, [_PS, _PS, _l, _l, _i, _i, _p, _p, _i, _i, _p, _i, _p, _p]),
    "pcb_proposal_epilogue": (_i, [_p, _i, _p, _l, _l, _i, _i, _f, _p, _p, _p, _p, _p]),
    "pcb_proposal_epilogue_grad": (_i, [_PS, _l, _l, _i, _i, _i, _f, _p, _p, _p, _p, _i, _i, _p, _p]),
    "pcb_voxel_down_sample_ws_bytes": (_sz, [_l, _l]),
    "pcb_voxel_down_sample": (_i, [_p, _l, _p, _l, _d, _p, _p, _p, _p, _sz, _p]),
    "pcb_frame_overlap_ws_bytes": (_sz, [_l, _l]),
    "pcb_frame_overlap": (_i, [_p, _l, _p, _l, _d, _p, _p, _p, _sz, _p]),
    "pcb_depth_to_points_ws_bytes": (_sz, [_l, _l, _l]),
    "pcb_depth_to_points": (_i, [_p, _l, _l, _l, _d, _d, _d, _d, _d, _d, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "pcb_nearest_ws_bytes": (_sz, [_l, _l]),
    "pcb_nearest": (_i, [_p, _l, _p, _l, _d, _p, _p, _p, _sz, _p]),
    "pcb_label_transfer": (_i, [_p, _p, _l, _p, _l, _p, _i, _i, _p, _p, _p, _p]),
    "pcb_text_lines_ws_bytes": (_sz, [_l]),
    "pcb_text_lines": (_i, [_p, _l, _p, C.c_int32, _p, _p, C.POINTER(C.c_int64), _p, _sz, _p]),
    "pcb_s3dis_parse": (_i, [_p, _l, _p, _p, C.c_int32, _p, _p, _l, _p, _p, _p, _p, _p, _p, _p]),
    "pcb_ply_rows": (_i, [_p, _p, _p, _p, _l, _p, _p]),
    "pcb_scannet_annotate_ws_bytes": (_sz, [_l, _l, _l]),
    "pcb_scannet_annotate": (_i, [_p, _p, _l, _p, _p, _p, _l, _p, _p, _l, _p, _p, _p, _l, _l, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "pcb_sunrgbd_votes": (_i, [_p, C.c_int32, _p, _p, _p, _p, _p, _l, _p, _p]),
}


class PcbTileDesc(C.Structure):
    """`struct pcb_tile_desc` of include/pcb200.h."""
    _fields_ = [("W", _p), ("fwd", _p), ("dgrad", _p), ("K", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32), ("flags", C.c_int32),
                ("bn_f", C.c_int32), ("bn_d", C.c_int32), ("start", _l)]


class PcbUnit(C.Structure):
    """`struct pcb_unit` of include/pcb200.h (field for field)."""
    _fields_ = [
        ("n_in", _l), ("n_out", _l), ("n0", _l),
        ("K", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32), ("relu", C.c_int32),
        ("fwd_tbl", _p), ("fwd_stride", _l), ("fwd_kmap", _p),
        ("dg_tbl", _p), ("dg_stride", _l), ("dg_kmap", _p),
        ("fwd_perm", _p),
        ("wg_tbl", _p), ("wg_stride", _l), ("wg_gather_x", C.c_int32),
        ("W", _p), ("wt_fwd", _p), ("wt_dg", _p), ("dW", _p),
        ("gamma", _p), ("beta", _p), ("running_mean", _p), ("running_var", _p), ("dgamma", _p), ("dbeta", _p),
        ("eps", _f), ("momentum", _f),
        ("mean", _p), ("invstd", _p),
        ("x_p", _p), ("x_ld", C.c_int32), ("x_hi", _p), ("x_lo", _p), ("x_lds", C.c_int32), ("x_bhi", _p), ("x_blo", _p),
        ("z_p", _p), ("z_ld", C.c_int32),
        ("out_p", _p), ("out_ld", C.c_int32), ("out_hi", _p), ("out_lo", _p), ("out_lds", C.c_int32), ("out_bhi", _p), ("out_blo", _p),
        ("res_p", _p), ("res_ld", C.c_int32),
        ("g_p", _p), ("g_ld", C.c_int32),
        ("dz_p", _p), ("dz_hi", _p), ("dz_lo", _p), ("dz_ld", C.c_int32),
        ("gin_p", _p), ("gin_ld", C.c_int32), ("gin_mode", C.c_int32),
        ("gres_p", _p), ("gres_ld", C.c_int32), ("gres_mode", C.c_int32),
        ("ws", _p), ("ws_bytes", _sz),
        ("flags", C.c_int32),
    ]
# Every integer `#define PCB_<NAME>` of include/pcb200.h as <NAME> (tests/test_host_abi.py holds this table to the header).
OK, ERR_CUDA, ERR_ARG = 0, 1, 2                       # return codes
ERR_RANGE, ERR_DUPLICATE = 3, 4                       # return codes, and the status bits of pcb_coords_pack / pcb_hash_build
MAX_KERNEL_VOLUME = 27
FRAMES_RANGE, FRAMES_OFFSETS = 1, 2                   # status bits of pcb_frame_overlap
NEAREST_RANGE, LABEL_RANGE = 1, 2                     # status bits of pcb_nearest / pcb_label_transfer
TEXT_NONASCII = 1                                     # file flag of pcb_text_lines
LINE_KEPT, LINE_SKIPPED, LINE_HOST, LINE_ERROR = 0, 1, 2, 3     # line status of pcb_s3dis_parse
CONV_FORCE_SIMT, CONV_ACCUMULATE = 1, 4               # flags of the convolution and weight-gradient entry points
PLANES_A_FP16, PLANES_B_FP16 = 8, 16                  # flags: 16-bit plane formats of the split-operand calls
BN_RELU = 1                                           # flag of pcb_bn_apply_seg
UNIT_SEPARATE_STATS, UNIT_FP16_FORWARD, UNIT_EVAL = 1, 2, 4     # pcb_unit.flags
DET_MAX_OBJ, DET_NPARAM = 64, 11                      # detection data: box slots per scene, params per scene
DET_SCANNET, DET_SUNRGBD = 0, 1                       # pcb_det_batch.dataset
DET_HEIGHT, DET_COLOR, DET_AUGMENT = 1, 2, 4          # pcb_det_batch.flags
EXPORTS = sorted(_SIGS)
for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)          # AttributeError here == the library does not export a declared symbol
    _fn.restype = _res
    _fn.argtypes = _args


def check(rc):
    if rc != 0:
        raise PcbError(f"libpcb200 error {rc}: {lib.pcb_last_error().decode()}")


def ptr(t):
    """Device (or None) pointer of a contiguous tensor."""
    if t is None:
        return None
    assert t.is_contiguous(), "libpcb200 needs contiguous tensors"
    return t.data_ptr()


_cur_dev = [-1]


def stream():
    """Current torch stream handle; also keeps the library's CUDA runtime on torch's current device."""
    d = torch.cuda.current_device()
    if d != _cur_dev[0]:
        check(lib.pcb_set_device(d))
        _cur_dev[0] = d
    return torch.cuda.current_stream().cuda_stream


_WS = {}


def workspace(nbytes, device):
    """Stream-ordered scratch owned by torch's allocator, one per (device, stream) and shared by every call on it (no entry point reads
    what an earlier call left in `ws`); grows, never shrinks.  Hold the tensor while its pointer is in use: a larger request replaces it."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    t = _WS.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.empty(max(int(nbytes), 1 << 20), dtype=torch.uint8, device=device)
        _WS[key] = t
    return t


def require_cuda(t):
    if not t.is_cuda:
        raise PcbError("pointcontrast_b200 ops run on CUDA tensors only (no CPU fallback); got a CPU tensor")


def launch_count():
    return int(lib.pcb_launch_count())
