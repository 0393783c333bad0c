"""ctypes binding of libumr_b200.so (C ABI declared in include/umr_b200.h).

The product path FAILS LOUDLY when the CUDA library is missing: there is no CPU fallback here
(the CPU oracle lives in oracle/ and is test infrastructure only).
"""
import ctypes
import os
import threading

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("UMR_B200_LIB") or os.path.join(_PKG, "libumr_b200.so")  # override: load another build, e.g. to compare two builds' outputs

c_f32p = ctypes.c_void_p  # raw device pointers are passed as integers (tensor.data_ptr())


class UmrRasterParams(ctypes.Structure):
    _fields_ = [("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32),
                ("texture_size", ctypes.c_int32), ("image_size", ctypes.c_int32),
                ("anti_aliasing", ctypes.c_int32),
                ("near_plane", ctypes.c_float), ("far_plane", ctypes.c_float), ("eps", ctypes.c_float),
                ("sigma_val", ctypes.c_float), ("dist_eps", ctypes.c_float), ("gamma_val", ctypes.c_float),
                ("func_id_dist", ctypes.c_int32), ("func_id_rgb", ctypes.c_int32),
                ("func_id_alpha", ctypes.c_int32), ("texture_sample_type", ctypes.c_int32),
                ("double_side", ctypes.c_int32), ("background_color", ctypes.c_float * 3),
                ("ev_kernel_start", ctypes.c_void_p), ("ev_kernel_stop", ctypes.c_void_p),
                ("pair_buffer", ctypes.c_void_p), ("pair_buffer_bytes", ctypes.c_uint64),
                ("shared_textures", ctypes.c_int32), ("tile_mode", ctypes.c_int32),
                ("color_channels", ctypes.c_int32), ("background_extra", ctypes.c_float)]


class UmrProjectParams(ctypes.Structure):
    _fields_ = [("batch_size", ctypes.c_int32), ("num_vertices", ctypes.c_int32), ("num_faces", ctypes.c_int32),
                ("flip_y", ctypes.c_int32), ("faces_batch_stride", ctypes.c_int64),
                ("offset_z", ctypes.c_float), ("eye_z", ctypes.c_float), ("viewing_scale", ctypes.c_float),
                ("light_enabled", ctypes.c_int32),
                ("light_intensity_ambient", ctypes.c_float), ("light_intensity_directional", ctypes.c_float),
                ("light_color_ambient", ctypes.c_float * 3), ("light_color_directional", ctypes.c_float * 3),
                ("light_direction", ctypes.c_float * 3), ("num_hypotheses", ctypes.c_int32)]


class UmrNmrParams(ctypes.Structure):
    _fields_ = [("batch_size", ctypes.c_int32), ("num_vertices", ctypes.c_int32), ("num_faces", ctypes.c_int32),
                ("texture_res", ctypes.c_int32), ("image_size", ctypes.c_int32), ("anti_aliasing", ctypes.c_int32),
                ("fill_back", ctypes.c_int32), ("shared_textures", ctypes.c_int32),
                ("eye_z", ctypes.c_float), ("near_plane", ctypes.c_float), ("far_plane", ctypes.c_float),
                ("light_intensity_ambient", ctypes.c_float), ("light_intensity_directional", ctypes.c_float),
                ("light_color_ambient", ctypes.c_float * 3), ("light_color_directional", ctypes.c_float * 3),
                ("light_direction", ctypes.c_float * 3), ("background_color", ctypes.c_float * 3)]


class UmrNmrLightParams(ctypes.Structure):
    _fields_ = [("batch_size", ctypes.c_int32), ("num_faces", ctypes.c_int32), ("texture_res", ctypes.c_int32),
                ("dtype", ctypes.c_int32), ("intensity_ambient", ctypes.c_double),
                ("intensity_directional", ctypes.c_double), ("color_ambient_bstride", ctypes.c_int32),
                ("color_directional_bstride", ctypes.c_int32), ("direction_bstride", ctypes.c_int32),
                ("reserved", ctypes.c_int32)]


EXPORTS = {
    # name: (restype, argtypes)
    "umr_error_string": (ctypes.c_char_p, [ctypes.c_int]),
    "umr_version": (ctypes.c_int, []),
    "umr_sizeof_raster_params": (ctypes.c_size_t, []),
    "umr_sizeof_project_params": (ctypes.c_size_t, []),
    "umr_launch_count": (ctypes.c_uint64, []),
    "umr_event_create": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p)]),
    "umr_event_destroy": (ctypes.c_int, [ctypes.c_void_p]),
    "umr_event_record": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "umr_event_elapsed_ms": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_float)]),
    "umr_raster_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 4),
    "umr_raster_pair_buffer_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3 + [ctypes.c_uint64]),
    "umr_raster_forward": (ctypes.c_int, [c_f32p] * 6 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                        ctypes.c_void_p]),
    "umr_raster_backward": (ctypes.c_int, [c_f32p] * 7 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                         ctypes.c_void_p]),
    "umr_raster_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 4),
    "umr_raster_forward_deterministic": (ctypes.c_int, [c_f32p] * 6 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                      ctypes.c_void_p]),
    "umr_raster_backward_deterministic": (ctypes.c_int, [c_f32p] * 7 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                       ctypes.c_void_p]),
    # split backward: alpha adjoint -> grad_faces, RGB adjoint -> grad_textures (the arguments of umr_raster_backward)
    "umr_raster_backward_split": (ctypes.c_int, [c_f32p] * 7 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                               ctypes.c_void_p]),
    "umr_raster_backward_split_deterministic": (ctypes.c_int, [c_f32p] * 7 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                             ctypes.c_void_p]),
    # silhouette render: alpha plane only (forward: face_vertices, alpha, alpha_hi; backward: face_vertices, alpha_hi,
    # grad_alpha, grad_faces)
    "umr_raster_forward_silhouette": (ctypes.c_int, [c_f32p] * 3 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                   ctypes.c_void_p]),
    "umr_raster_forward_silhouette_deterministic": (ctypes.c_int, [c_f32p] * 3 + [ctypes.POINTER(UmrRasterParams),
                                                                                 ctypes.c_void_p, ctypes.c_void_p]),
    "umr_raster_backward_silhouette": (ctypes.c_int, [c_f32p] * 4 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                    ctypes.c_void_p]),
    "umr_raster_backward_silhouette_deterministic": (ctypes.c_int, [c_f32p] * 4 + [ctypes.POINTER(UmrRasterParams),
                                                                                  ctypes.c_void_p, ctypes.c_void_p]),
    # double-precision rasteriser: the arguments of umr_raster_forward / umr_raster_backward with double buffers
    "umr_raster_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32] * 4),
    "umr_raster_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                     ctypes.c_void_p]),
    "umr_raster_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 7 + [ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                                                      ctypes.c_void_p]),
    "umr_raster_visibility": (ctypes.c_int, [c_f32p, c_f32p, ctypes.c_void_p, ctypes.POINTER(UmrRasterParams), ctypes.c_void_p,
                                             ctypes.c_void_p]),
    "umr_corr_chamfer_forward": (ctypes.c_int, [c_f32p, ctypes.c_int64, c_f32p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p),
                                                ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32),
                                                ctypes.POINTER(ctypes.c_float), c_f32p, ctypes.c_void_p, c_f32p, ctypes.c_int32,
                                                ctypes.c_int32, ctypes.c_void_p]),
    "umr_corr_chamfer_backward": (ctypes.c_int, [c_f32p, ctypes.c_int64, c_f32p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p),
                                                 ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32),
                                                 ctypes.POINTER(ctypes.c_float), c_f32p, ctypes.c_void_p, c_f32p, c_f32p, c_f32p,
                                                 c_f32p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p]),
    "umr_project_faces_forward": (ctypes.c_int, [c_f32p] * 5 + [ctypes.POINTER(UmrProjectParams), ctypes.c_void_p]),
    "umr_project_faces_backward": (ctypes.c_int, [c_f32p] * 8 + [ctypes.POINTER(UmrProjectParams), ctypes.c_void_p]),
    "umr_bilinear_sample_forward": (ctypes.c_int, [c_f32p] * 3 + [ctypes.c_int32] * 5 + [ctypes.c_void_p]),
    "umr_bilinear_sample_backward": (ctypes.c_int, [c_f32p] * 5 + [ctypes.c_int32] * 5 + [ctypes.c_void_p]),
    "umr_iou_forward": (ctypes.c_int, [c_f32p, ctypes.c_int64] + [c_f32p] * 4 + [ctypes.c_int32, ctypes.c_int64,
                                                                                  ctypes.c_void_p]),
    "umr_iou_backward": (ctypes.c_int, [c_f32p] * 5 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p]),
    "umr_masked_l1_forward": (ctypes.c_int, [c_f32p, ctypes.c_int64, c_f32p, ctypes.c_int64, c_f32p, c_f32p, c_f32p,
                                             ctypes.c_int32, ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p]),
    "umr_masked_l1_backward": (ctypes.c_int, [c_f32p, ctypes.c_int64, c_f32p, ctypes.c_int64, c_f32p, c_f32p, c_f32p,
                                              c_f32p, c_f32p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int64,
                                              ctypes.c_void_p]),
    "umr_loss_head_forward": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_float,
                                                     ctypes.c_void_p]),
    "umr_loss_head_backward": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_float,
                                                      ctypes.c_void_p]),
    "umr_create_texture_image": (ctypes.c_int, [c_f32p] * 3 + [ctypes.c_int32] * 4 + [ctypes.c_float, ctypes.c_void_p]),
    "umr_load_textures": (ctypes.c_int, [c_f32p] * 4 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_laplacian_forward": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 2 + [ctypes.c_void_p]),
    "umr_laplacian_backward": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 2 + [ctypes.c_void_p]),
    "umr_flatten_forward": (ctypes.c_int, [c_f32p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_float, ctypes.c_void_p]),
    "umr_flatten_backward": (ctypes.c_int, [c_f32p] * 4 + [ctypes.c_int32] * 3 + [ctypes.c_float, ctypes.c_void_p]),
    "umr_dt_barrier_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "umr_dt_barrier": (ctypes.c_int, [c_f32p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_float, ctypes.c_void_p]),
    "umr_p2p_allreduce_flag_bytes": (ctypes.c_size_t, []),
    "umr_p2p_allreduce": (ctypes.c_int, [ctypes.c_void_p, c_f32p, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int32,
                                         ctypes.c_int32, ctypes.c_float, ctypes.c_void_p]),
    "umr_chamfer_forward": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_chamfer_backward": (ctypes.c_int, [c_f32p] * 8 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_texcycle_forward": (ctypes.c_int, [c_f32p] * 5 + [ctypes.c_int32] * 3 + [ctypes.c_int64,
                                                                                ctypes.c_void_p]),
    "umr_texcycle_backward": (ctypes.c_int, [c_f32p] * 5 + [ctypes.c_int32] * 3 + [ctypes.c_void_p]),
    "umr_sizeof_nmr_params": (ctypes.c_size_t, []),
    "umr_nmr_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "umr_nmr_forward": (ctypes.c_int, [c_f32p] * 8 + [ctypes.POINTER(UmrNmrParams), ctypes.c_void_p, ctypes.c_void_p]),
    "umr_nmr_backward_textures": (ctypes.c_int, [c_f32p] * 5 + [ctypes.POINTER(UmrNmrParams), ctypes.c_void_p,
                                                                ctypes.c_void_p]),
    # geometry gradient of the functional rasteriser: vertices, faces, face_index, textures, grad_rgb, grad_alpha,
    # grad_depth, grad_face_vertices, params, eps, workspace, stream
    "umr_nmr_backward_faces_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 4),
    "umr_nmr_backward_faces": (ctypes.c_int, [c_f32p] * 8 + [ctypes.POINTER(UmrNmrParams), ctypes.c_float, ctypes.c_void_p,
                                                             ctypes.c_void_p]),
    # neural_renderer.lighting: faces, textures, color_ambient, color_directional, direction, lit_textures (forward);
    # ..., grad_lit, grad_faces, grad_textures, grad_light, params, workspace, stream (backward)
    "umr_sizeof_nmr_light_params": (ctypes.c_size_t, []),
    "umr_nmr_lighting_forward": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.POINTER(UmrNmrLightParams), ctypes.c_void_p]),
    "umr_nmr_lighting_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "umr_nmr_lighting_backward": (ctypes.c_int, [ctypes.c_void_p] * 9 + [ctypes.POINTER(UmrNmrLightParams), ctypes.c_void_p,
                                                                        ctypes.c_void_p]),
    "umr_voxelize_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_voxelize": (ctypes.c_int, [c_f32p, ctypes.c_int32, c_f32p] + [ctypes.c_int32] * 3 + [ctypes.c_double, ctypes.c_void_p,
                                                                                           ctypes.c_void_p]),
    # deterministic loss kernels: the default symbol's arguments + a workspace (+ the transposed tables of flatten / corr)
    "umr_iou_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "umr_iou_forward_deterministic": (ctypes.c_int, [c_f32p, ctypes.c_int64] + [c_f32p] * 4 + [ctypes.c_int32, ctypes.c_int64,
                                                                                                ctypes.c_void_p, ctypes.c_void_p]),
    "umr_masked_l1_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "umr_masked_l1_forward_deterministic": (ctypes.c_int, [c_f32p, ctypes.c_int64, c_f32p, ctypes.c_int64, c_f32p, c_f32p, c_f32p,
                                                           ctypes.c_int32, ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p,
                                                           ctypes.c_void_p]),
    "umr_loss_head_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "umr_loss_head_forward_deterministic": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_float,
                                                                   ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]),
    "umr_texcycle_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_texcycle_forward_deterministic": (ctypes.c_int, [c_f32p] * 5 + [ctypes.c_int32] * 3 + [ctypes.c_int64, ctypes.c_void_p,
                                                                                              ctypes.c_void_p]),
    "umr_laplacian_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_laplacian_forward_deterministic": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 2 + [ctypes.c_void_p, ctypes.c_void_p]),
    "umr_flatten_forward_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_flatten_forward_deterministic": (ctypes.c_int, [c_f32p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_float, ctypes.c_void_p,
                                                                                             ctypes.c_void_p]),
    "umr_flatten_backward_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_flatten_backward_deterministic": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 3 + [ctypes.c_float, ctypes.c_void_p,
                                                                                              ctypes.c_void_p]),
    "umr_chamfer_backward_deterministic": (ctypes.c_int, [c_f32p] * 8 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_corr_chamfer_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_corr_chamfer_backward_deterministic": (ctypes.c_int, [c_f32p, ctypes.c_int64, c_f32p, ctypes.c_void_p,
                                                               ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int32),
                                                               ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_float),
                                                               c_f32p, ctypes.c_void_p, c_f32p, c_f32p, c_f32p, c_f32p,
                                                               ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    # deterministic vertex / NMR texture / sampler image backwards (+ the device-built transposed tables)
    "umr_project_faces_workspace_bytes_deterministic": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "umr_project_faces_backward_deterministic": (ctypes.c_int, [c_f32p] * 8 + [ctypes.POINTER(UmrProjectParams)] +
                                                 [ctypes.c_void_p] * 4),
    "umr_nmr_backward_textures_deterministic": (ctypes.c_int, [c_f32p] * 5 + [ctypes.POINTER(UmrNmrParams), ctypes.c_void_p,
                                                                              ctypes.c_void_p]),
    "umr_bilinear_sample_cells": (ctypes.c_int, [c_f32p, ctypes.c_void_p] + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_bilinear_sample_backward_deterministic": (ctypes.c_int, [c_f32p] * 5 + [ctypes.c_int32] * 5 + [ctypes.c_void_p] * 3),
    # float64 loss kernels: the float32 symbol's arguments with double buffers / scalars (+ a workspace for reductions)
    "umr_bilinear_sample_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 5 + [ctypes.c_void_p]),
    "umr_bilinear_sample_cells_f64": (ctypes.c_int, [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_bilinear_sample_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int32] * 5 + [ctypes.c_void_p] * 3),
    "umr_iou_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "umr_iou_forward_f64": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 4 +
                            [ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "umr_iou_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p]),
    "umr_masked_l1_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "umr_masked_l1_forward_f64": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64] +
                                  [ctypes.c_void_p] * 3 + [ctypes.c_int32, ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p,
                                                           ctypes.c_void_p]),
    "umr_masked_l1_backward_f64": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64] +
                                   [ctypes.c_void_p] * 5 + [ctypes.c_int32, ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p]),
    "umr_loss_head_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "umr_loss_head_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_double,
                                                                         ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]),
    "umr_loss_head_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int32, ctypes.c_int64, ctypes.c_double,
                                                                          ctypes.c_double, ctypes.c_void_p]),
    "umr_chamfer_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_chamfer_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 8 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
    "umr_texcycle_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_texcycle_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int32] * 3 + [ctypes.c_int64, ctypes.c_void_p,
                                                                                               ctypes.c_void_p]),
    "umr_texcycle_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int32] * 3 + [ctypes.c_void_p]),
    "umr_laplacian_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_laplacian_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 2),
    "umr_laplacian_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int32] * 2 + [ctypes.c_void_p]),
    "umr_flatten_forward_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_flatten_forward_f64": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_double, ctypes.c_void_p,
                                                                                              ctypes.c_void_p]),
    "umr_flatten_backward_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_flatten_backward_f64": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int32] * 3 + [ctypes.c_double, ctypes.c_void_p,
                                                                                               ctypes.c_void_p]),
    "umr_corr_chamfer_forward_f64": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                                    ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int32),
                                                    ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_double)] +
                                     [ctypes.c_void_p] * 3 + [ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p]),
    "umr_corr_chamfer_workspace_bytes_f64": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "umr_corr_chamfer_backward_f64": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                                     ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int32),
                                                     ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_double)] +
                                      [ctypes.c_void_p] * 6 + [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 4),
    # part_matching_loss head: maps / map_bstrides are host arrays of 4; `dtype` as umr_voxelize takes it
    "umr_part_head_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "umr_part_head_forward": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int64), ctypes.c_void_p,
                                             ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p] +
                              [ctypes.c_int32] * 4 + [ctypes.c_void_p] * 2),
    "umr_part_head_backward": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int64), ctypes.c_void_p,
                                              ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 4 +
                               [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
}

# Keypoint transfer of the keypoint evaluation (include/umr_kp_transfer.h), bound by load() like EXPORTS.  A table of its
# own, as the header is: EXPORTS lists umr_b200.h's own declarations.
KP_EXPORTS = {
    # kps, flow_src, flow_tgt, gauss, grid, out, P, K, F, T2, S, sigma, stream
    "umr_kp_transfer_flow": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 6 + [ctypes.c_void_p]),
    # kps, proj_src, proj_tgt, mask_tgt, grid, out, P, K, V, S, stream
    "umr_kp_transfer_cam": (ctypes.c_int, [c_f32p] * 6 + [ctypes.c_int32] * 4 + [ctypes.c_void_p]),
}

# SCOPS part centres and part points (include/umr_part_points.h), bound by load() like EXPORTS, in a table of its own as
# KP_EXPORTS is.
PP_EXPORTS = {
    # part_prob, mask, uniforms, B, S, C, K, channels, num_samples (host int32 [K]), dtype, centers_in, centers,
    # points, drawn (host pointer arrays [K]), status, stream
    "umr_part_points": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 4 +
                        [ctypes.POINTER(ctypes.c_int32)] * 2 + [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p] +
                        [ctypes.POINTER(ctypes.c_void_p)] * 2 + [ctypes.c_void_p, ctypes.c_void_p]),
}

# SCOPS semantic template (include/umr_semantic_template.h), bound by load() like EXPORTS, in a table of its own as
# KP_EXPORTS is.
ST_EXPORTS = {
    # B, H, W
    "umr_st_average_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    # part_segs, uvimage_pred, exemplar, B, C, S, H, W, k, workspace, dist, selected, acc, stream
    "umr_st_average_add": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 6 + [ctypes.c_void_p] * 5),
    # acc, C, H, W, count, avg_prob, stream
    "umr_st_average_mean": (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int32] * 3 + [ctypes.c_int64, ctypes.c_void_p,
                                                                                       ctypes.c_void_p]),
    # avg_prob, H, W, C, uv_sampler, F_src, T2, num_sym_faces, vertex_rowptr, vertex_corners, V, label_image,
    # texel_labels, face_labels, vertex_labels, stream
    "umr_st_labels": (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int32] * 3 + [ctypes.c_void_p] + [ctypes.c_int32] * 3 +
                      [ctypes.c_void_p] * 2 + [ctypes.c_int32] + [ctypes.c_void_p] * 5),
}

# Training batch crop / resize / mirror / normalisation (include/umr_crop.h), bound by load() like EXPORTS, in a table
# of its own as KP_EXPORTS is.
CROP_EXPORTS = {
    # pack, pack_bytes, table_dev, table_host, B, S, part_prob, C, imgs, input_imgs, masks, part_prob_out, part_segs,
    # stream
    "umr_crop_batch": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32),
                                      ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32] +
                       [ctypes.c_void_p] * 6),
}

_lock = threading.Lock()
_lib = None


class UmrLibraryError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises UmrLibraryError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise UmrLibraryError(
                    "libumr_b200.so is not built (%s). Run `python -m umr_b200.build` "
                    "(or __graft_entry__.build()). There is no CPU fallback." % LIB_PATH)
            lib = ctypes.CDLL(LIB_PATH)
            for name, (res, args) in list(EXPORTS.items()) + list(KP_EXPORTS.items()) + list(PP_EXPORTS.items()) + \
                    list(ST_EXPORTS.items()) + list(CROP_EXPORTS.items()):
                fn = getattr(lib, name)  # AttributeError if the symbol is missing
                fn.restype = res
                fn.argtypes = args
            if (lib.umr_sizeof_raster_params() != ctypes.sizeof(UmrRasterParams)
                    or lib.umr_sizeof_project_params() != ctypes.sizeof(UmrProjectParams)
                    or lib.umr_sizeof_nmr_params() != ctypes.sizeof(UmrNmrParams)
                    or lib.umr_sizeof_nmr_light_params() != ctypes.sizeof(UmrNmrLightParams)):
                raise UmrLibraryError("libumr_b200.so was built from a different include/umr_b200.h than this binding "
                                      "(parameter struct sizes differ): rebuild with `python -m umr_b200.build --force`")
            _lib = lib
    return _lib


def check(code, what):
    if code != 0:
        msg = load().umr_error_string(int(code))
        raise RuntimeError("%s failed: %s (code %d)" % (what, msg.decode() if msg else "?", code))
