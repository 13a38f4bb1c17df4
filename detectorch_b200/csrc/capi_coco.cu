// detectorch_b200 -- C-ABI entry points of the COCO evaluation (coco_eval.cuh), the results json (coco_json.cuh) and the proposal
// recall (proposal_recall.cuh); include/detectorch_b200.h.
#include <stdio.h>

#include "../../include/detectorch_b200.h"
#include "coco_eval.cuh"
#include "coco_json.cuh"
#include "coco_results_file.cuh"
#include "common.cuh"
#include "proposal_recall.cuh"

using namespace dt;

extern "C" int64_t dt_coco_gt_workspace_bytes(int64_t num_parts, int64_t num_points, int64_t num_upsampled) {
    if (num_parts < 0 || num_points < 0 || num_upsampled < 0) return 0;
    return 4 * (num_points + 4 * num_upsampled + 3 * num_parts);
}

extern "C" int dt_coco_gt_build(int num_anns, const int64_t* anns, const int64_t* parts, const double* xy, const uint32_t* ucounts,
                                const char* chars, void* workspace, uint32_t* out_counts, uint32_t* tmp_counts, int64_t* out_len,
                                double* out_box, dt_stream_t stream) {
    if (num_anns < 0) { fprintf(stderr, "dt_coco_gt_build: negative annotation count\n"); return 0; }
    if (num_anns == 0) return 1;
    if (!anns || !parts || !out_counts || !tmp_counts || !out_len || !out_box) {
        fprintf(stderr, "dt_coco_gt_build: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(coco_gt_launch(num_anns, anns, parts, xy, ucounts, chars, reinterpret_cast<int*>(workspace), out_counts, tmp_counts,
                                 out_len, out_box, (cudaStream_t)stream));
    return 1;
}

extern "C" int dt_coco_det_check(int64_t num_dets, const int64_t* det_i, const char* det_chars, uint8_t* bad, dt_stream_t stream) {
    if (num_dets < 0) { fprintf(stderr, "dt_coco_det_check: negative detection count\n"); return 0; }
    if (num_dets == 0) return 1;
    if (!det_i || !det_chars || !bad) { fprintf(stderr, "dt_coco_det_check: null argument\n"); return 0; }
    DT_CHECK_CUDA(coco_det_check_launch(num_dets, det_i, det_chars, bad, (cudaStream_t)stream));
    return 1;
}

extern "C" int64_t dt_coco_eval_workspace_bytes(int64_t num_dets, int64_t num_chars, int64_t kept, int64_t num_ious, int64_t num_gts,
                                                int64_t num_order, int num_cats) {
    if (num_dets < 0 || num_chars < 0 || kept < 0 || num_ious < 0 || num_gts < 0 || num_order < 0 || num_cats < 0 ||
        kCocoMaxDets * kept >= (1ll << 31))
        return 0;
    return (int64_t)coco_eval_ws(num_dets, num_chars, kept, num_ious, num_gts, num_order, num_cats).total_with_rank;
}

extern "C" int dt_coco_eval(int iou_type, int num_images, int num_cats, int num_active, const int64_t* pairs, const int64_t* cat_gt,
                            const int64_t* cat_kept, const int64_t* order_off, int64_t num_dets, const double* det_f, const int64_t* det_i,
                            const char* det_chars, int64_t num_chars, int64_t kept, int64_t num_ious, int64_t num_gts, int64_t num_order,
                            const double* gt_f, const int64_t* gt_i, const uint32_t* gt_counts, const double* params, double* precision,
                            double* recall, double* scores, double* ious, void* workspace, dt_stream_t stream, const double* det_area) {
    if ((iou_type != 0 && iou_type != 1) || num_images < 0 || num_cats < 0 || num_active < 0 || num_dets < 0 || num_chars < 0 || kept < 0 ||
        num_ious < 0 || num_gts < 0 || num_order < 0 || kept > num_dets || num_active > num_dets || (int64_t)num_cats * 120 >= (1ll << 31) ||
        kCocoMaxDets * kept >= (1ll << 31)) {
        fprintf(stderr, "dt_coco_eval: bad sizes\n");
        return 0;
    }
    if (num_cats == 0) return 1;
    if (!cat_gt || !cat_kept || !order_off || !params || !precision || !recall || !scores || (num_gts > 0 && (!gt_f || !gt_i)) ||
        (iou_type == 1 && num_gts > 0 && !gt_counts) || (num_dets > 0 && (!pairs || !det_f || !det_i || !workspace)) ||
        (iou_type == 1 && num_chars > 0 && !det_chars)) {
        fprintf(stderr, "dt_coco_eval: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(coco_eval_launch(iou_type, num_images, num_cats, num_active, pairs, cat_gt, cat_kept, order_off, num_dets, det_f, det_i,
                                   det_chars, num_chars, kept, num_ious, num_gts, num_order, gt_f, gt_i, gt_counts, params, precision, recall,
                                   scores, ious, workspace, (cudaStream_t)stream, det_area));
    return 1;
}

extern "C" int dt_coco_eval_imgs(int iou_type, int num_union, const int64_t* union_keys, int num_active, const int64_t* pairs, int64_t num_dets,
                                 const double* det_f, int64_t num_chars, int64_t kept, int64_t num_ious, int64_t num_gts, int64_t num_order,
                                 const int64_t* gt_keys, const double* gt_f, const int64_t* gt_i, const double* params, const double* ious,
                                 const void* workspace, int* slot_det, int* dt_gt, uint8_t* dt_ig, int* gt_dt, int* gt_pos, uint8_t* gt_ig,
                                 dt_stream_t stream, const double* det_area) {
    if ((iou_type != 0 && iou_type != 1) || num_union < 0 || num_active < 0 || num_dets < 0 || num_chars < 0 || kept < 0 || num_ious < 0 ||
        num_gts < 0 || num_order < 0 || kept > num_dets || num_active > num_dets || num_active > num_union) {
        fprintf(stderr, "dt_coco_eval_imgs: bad sizes\n");
        return 0;
    }
    if (num_union == 0) return 1;
    if (!union_keys || !params || (num_gts > 0 && (!gt_keys || !gt_f || !gt_i || !gt_dt || !gt_pos || !gt_ig)) ||
        (num_active > 0 && (!pairs || !det_f || !ious || !workspace || !slot_det || !dt_gt || !dt_ig))) {
        fprintf(stderr, "dt_coco_eval_imgs: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(coco_eval_imgs_launch(iou_type, num_union, union_keys, num_active, pairs, num_dets, num_chars, kept, num_ious, num_gts, num_order,
                                        gt_keys, det_f, gt_f, gt_i, params, ious, workspace, slot_det, dt_gt, dt_ig, gt_dt, gt_pos, gt_ig,
                                        (cudaStream_t)stream, det_area));
    return 1;
}

extern "C" int dt_coco_results_append(int batch, int cap, int num_classes, const float* boxes, const float* scores, const int* classes,
                                      const int* counts, const int64_t* images, const int64_t* str_offs, int64_t char_base, float* rec_f,
                                      int64_t* rec_i, int* err, dt_stream_t stream) {
    if (batch < 0 || cap < 0 || num_classes < 1 || char_base < 0) { fprintf(stderr, "dt_coco_results_append: bad sizes\n"); return 0; }
    if ((int64_t)batch * cap == 0) return 1;
    if (!boxes || !scores || !classes || !counts || !images || !rec_f || !rec_i || !err) {
        fprintf(stderr, "dt_coco_results_append: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(coco_results_append_launch(batch, cap, num_classes, boxes, scores, classes, counts, images, str_offs, char_base, rec_f, rec_i,
                                             err, (cudaStream_t)stream));
    return 1;
}

extern "C" int dt_coco_results_count(int64_t num_records, const float* rec_f, const int64_t* rec_i, int num_classes, const int* cls_k,
                                     const int* ord_i, int num_images, int num_cats, int cats_per_pair, const int64_t* gt_keys, int64_t num_gts,
                                     int* bin_cnt, int64_t* scan_in, int* nonfinite, dt_stream_t stream) {
    if (num_records < 0 || num_classes < 1 || num_images < 0 || num_cats < 0 || num_gts < 0 || cats_per_pair < 1 ||
        (cats_per_pair > 1 && num_cats != 1)) {
        fprintf(stderr, "dt_coco_results_count: bad sizes\n");
        return 0;
    }
    if ((num_records > 0 && (!rec_f || !rec_i || !cls_k || !ord_i || !nonfinite)) ||
        ((int64_t)num_images * num_cats > 0 && (!bin_cnt || !scan_in || (num_gts > 0 && !gt_keys)))) {
        fprintf(stderr, "dt_coco_results_count: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(coco_results_count_launch(num_records, rec_f, rec_i, num_classes, cls_k, ord_i, num_images, num_cats, cats_per_pair, gt_keys,
                                            num_gts, bin_cnt, scan_in, nonfinite, (cudaStream_t)stream));
    return 1;
}

extern "C" int dt_coco_results_write(int64_t num_records, const float* rec_f, const int64_t* rec_i, int num_classes, const int* cls_k,
                                     const int* ord_i, int num_images, int num_cats, int cats_per_pair, const int* bin_cnt, const int64_t* scan,
                                     const int64_t* gt_keys, int64_t num_gts, int64_t* det_key, double* det_f, int64_t* det_i, int64_t* pairs,
                                     int64_t* cat_kept, int64_t* order_off, dt_stream_t stream) {
    if (num_records < 0 || num_classes < 1 || num_images < 0 || num_cats < 0 || num_gts < 0 || cats_per_pair < 1 ||
        (cats_per_pair > 1 && num_cats != 1)) {
        fprintf(stderr, "dt_coco_results_write: bad sizes\n");
        return 0;
    }
    const bool bins = (int64_t)num_images * num_cats > 0;
    if ((num_records > 0 && (!rec_f || !rec_i || !cls_k || !ord_i || (bins && (!det_key || !det_f || !det_i)))) || !cat_kept || !order_off ||
        (bins && (!scan || !bin_cnt || (num_gts > 0 && !gt_keys)))) {
        fprintf(stderr, "dt_coco_results_write: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(coco_results_write_launch(bins ? num_records : 0, rec_f, rec_i, num_classes, cls_k, ord_i, num_images, num_cats, cats_per_pair,
                                            bin_cnt, scan, gt_keys, num_gts, det_key, det_f, det_i, pairs, cat_kept, order_off, (cudaStream_t)stream));
    return 1;
}

extern "C" int dt_coco_json(int iou_type, int64_t num_dets, const double* det_f, const int64_t* det_key, const int64_t* file_pos, int num_images,
                            const int64_t* img_ids, const int64_t* cat_ids, const int64_t* det_i, const char* det_chars,
                            const uint8_t* counts_first, const int64_t* offsets, int64_t* lens, char* text, dt_stream_t stream) {
    if ((iou_type != 0 && iou_type != 1) || num_dets < 0 || num_images < 0 || (num_dets > 0 && num_images == 0) ||
        num_dets > (1ll << 31) / 32) {
        fprintf(stderr, "dt_coco_json: bad sizes\n");
        return 0;
    }
    if (num_dets == 0) return 1;
    if (!det_f || !det_key || !file_pos || !img_ids || !cat_ids || (iou_type == 1 && (!det_i || !det_chars)) || (offsets ? !text : !lens)) {
        fprintf(stderr, "dt_coco_json: null argument\n");
        return 0;
    }
    JsonRows R{num_dets, num_images, det_f, det_key, file_pos, img_ids, cat_ids, det_i, det_chars, counts_first};
    DT_CHECK_CUDA(coco_json_launch(iou_type, R, offsets, lens, text, (cudaStream_t)stream));
    return 1;
}

extern "C" int64_t dt_coco_file_struct_workspace_bytes(int64_t num_bytes) {
    if (num_bytes < 1) return 0;
    return (int64_t)cf_struct_ws(num_bytes).total;
}

extern "C" int dt_coco_file_struct(int64_t num_bytes, const uint8_t* text, void* workspace, int64_t* info, dt_stream_t stream) {
    if (num_bytes < 1) { fprintf(stderr, "dt_coco_file_struct: empty text\n"); return 0; }
    if (!text || !workspace || !info) { fprintf(stderr, "dt_coco_file_struct: null argument\n"); return 0; }
    DT_CHECK_CUDA(cf_struct_launch(num_bytes, text, reinterpret_cast<uint8_t*>(workspace), reinterpret_cast<unsigned long long*>(info),
                                   (cudaStream_t)stream));
    return 1;
}

extern "C" int dt_coco_file_separators(int64_t num_bytes, void* workspace, int64_t* separators, dt_stream_t stream) {
    if (num_bytes < 1) { fprintf(stderr, "dt_coco_file_separators: empty text\n"); return 0; }
    if (!workspace || !separators) { fprintf(stderr, "dt_coco_file_separators: null argument\n"); return 0; }
    DT_CHECK_CUDA(cf_separators_launch(num_bytes, reinterpret_cast<uint8_t*>(workspace), separators, (cudaStream_t)stream));
    return 1;
}

extern "C" int dt_coco_file_records(int64_t num_records, int64_t num_bytes, const uint8_t* text, const int64_t* separators, int num_images,
                                    const int64_t* img_ids, int num_cats, const int64_t* cat_ids, double* rec_f, int64_t* rec_open, int64_t* rec_i,
                                    int64_t* rec_n, uint8_t* rec_b, int64_t* info, dt_stream_t stream) {
    if (num_records < 0 || num_bytes < 1 || num_images < 0 || num_cats < 0) { fprintf(stderr, "dt_coco_file_records: bad sizes\n"); return 0; }
    if (num_records == 0) return 1;
    if (!text || !separators || (num_images > 0 && !img_ids) || (num_cats > 0 && !cat_ids) || !rec_f || !rec_open || !rec_i || !rec_n || !rec_b ||
        !info) {
        fprintf(stderr, "dt_coco_file_records: null argument\n");
        return 0;
    }
    CfArgs a{num_records, text, separators, num_images, num_cats, img_ids, cat_ids, rec_f, rec_open, rec_i, rec_n, rec_b,
             reinterpret_cast<unsigned long long*>(info)};
    DT_CHECK_CUDA(cf_records_launch(a, num_bytes, (cudaStream_t)stream));
    return 1;
}

extern "C" int64_t dt_coco_file_finish_workspace_bytes(int64_t num_records, int64_t num_chars, int segm) {
    if (num_records < 1 || num_chars < 0) return 0;
    return (int64_t)cf_finish_ws(num_records, num_chars, segm).total;
}

extern "C" int dt_coco_file_finish(int64_t num_records, int segm, const uint8_t* text, const int64_t* rec_i, const int64_t* rec_n,
                                   const int64_t* offsets, const uint8_t* rec_b, double* rec_f, int num_images, int num_cats, int64_t num_chars,
                                   char* chars, void* workspace, int64_t num_kept, int64_t* det_key, double* det_f, int64_t* det_i,
                                   double* det_area, int64_t* det_id, int64_t* info, dt_stream_t stream) {
    if (num_records < 1 || num_images < 0 || num_cats < 0 || num_chars < 0 || num_kept < 0 || num_kept > num_records) {
        fprintf(stderr, "dt_coco_file_finish: bad sizes\n");
        return 0;
    }
    if (!text || !rec_i || !rec_n || !offsets || !rec_b || !rec_f || !chars || !workspace || !det_key || !info ||
        (num_kept > 0 && (!det_f || !det_i || !det_area || !det_id))) {
        fprintf(stderr, "dt_coco_file_finish: null argument\n");
        return 0;
    }
    DT_CHECK_CUDA(cf_finish_launch(num_records, segm, text, rec_i, rec_n, offsets, rec_b, rec_f, num_images, num_cats, num_chars, chars,
                                   reinterpret_cast<uint8_t*>(workspace), num_kept, det_key, det_f, det_i, det_area, det_id,
                                   reinterpret_cast<unsigned long long*>(info), (cudaStream_t)stream));
    return 1;
}

extern "C" int64_t dt_proposal_recall_smem_bytes(int max_gts, int64_t max_props) {
    if (max_gts < 0 || max_props < 0 || max_gts > (1 << 24) || max_props > (1ll << 36)) return 0;
    return (int64_t)proposal_recall_smem(max_gts, (int)((max_props + 31) / 32));
}

extern "C" int dt_proposal_recall(int num_images, int num_combos, const int64_t* prop_off, const float* props, const int64_t* gt_off,
                                  const float* gts, const double* gt_area, const double* area_rng, const int64_t* limits,
                                  const int64_t* out_off, int max_gts, int64_t max_props, double* out, int* flag, dt_stream_t stream) {
    if (num_images < 0 || num_combos < 0 || num_combos > 65535 || max_gts < 0 || max_props < 0 || max_props > (1ll << 36)) {
        fprintf(stderr, "dt_proposal_recall: bad sizes\n");
        return 0;
    }
    if (num_images == 0 || num_combos == 0) return 1;
    if (!prop_off || !gt_off || !area_rng || !limits || !out_off || !flag || (max_props > 0 && !props) || (max_gts > 0 && (!gts || !gt_area || !out))) {
        fprintf(stderr, "dt_proposal_recall: null argument\n");
        return 0;
    }
    const int words = (int)((max_props + 31) / 32);
    if (proposal_recall_smem(max_gts, words) > 227 * 1024) {
        fprintf(stderr, "dt_proposal_recall: %d ground-truth boxes and %lld proposals in one image exceed shared memory\n", max_gts,
                (long long)max_props);
        return 0;
    }
    if (max_gts == 0) return 1;
    RecallParams P;
    P.num_images = num_images;
    P.prop_off = prop_off; P.props = reinterpret_cast<const float4*>(props);
    P.gt_off = gt_off; P.gts = reinterpret_cast<const float4*>(gts); P.gt_area = gt_area;
    P.area_rng = area_rng; P.limits = limits; P.out_off = out_off; P.out = out; P.flag = flag;
    P.max_gts = max_gts; P.row_words = words;
    DT_CHECK_CUDA(proposal_recall_launch(P, num_combos, (cudaStream_t)stream));
    return 1;
}
