"""Host restatement of WaymoDataset.convert_valid_bboxes / bbox2result_kitti (mmdet3d
datasets/waymo_dataset.py) for load_mode 'lidar_frame', one frame at a time on CPU float32
tensors with the same torch / numpy operations as the reference's box structures.  It is the
reference the device conversion (``dfm_waymo_kitti_convert``) is checked against.

The rules that differ from KittiDataset's:
- camera boxes always come from R0_rect @ Tr_velo_to_cam (float32), and corners are
  projected with P0, not P2;
- a box is kept iff its centre lies strictly inside pcd_limit_range; there is no image test;
- a frame that keeps nothing has label_preds of shape [0] and writes no submission file;
- submission files are named <sample_idx:07d>.txt.
"""
import os

import numpy as np

from depth_from_motion_b200.kitti_eval import (_boxes_tensor, _cam_corners, _limit_period,
                                               _lidar_to_cam, _points_cam2img)

WAYMO_PCD_LIMIT_RANGE = (-85, -85, -5, 85, 85, 5)


def convert_valid_bboxes(box_dict, info, pcd_limit_range=WAYMO_PCD_LIMIT_RANGE):
    import torch
    t = _boxes_tensor(box_dict['boxes_3d'])
    scores = torch.as_tensor(box_dict['scores_3d']).detach().cpu()
    labels = torch.as_tensor(box_dict['labels_3d']).detach().cpu()
    sample_idx = info['image']['image_idx']
    t[:, 6] = _limit_period(t[:, 6], 0.5, np.pi * 2)
    empty = dict(bbox=np.zeros([0, 4]), box3d_camera=np.zeros([0, 7]),
                 box3d_lidar=np.zeros([0, 7]), scores=np.zeros([0]),
                 label_preds=np.zeros([0]), sample_idx=sample_idx)
    if len(t) == 0:
        return empty
    rect = info['calib']['R0_rect'].astype(np.float32)
    Trv2c = info['calib']['Tr_velo_to_cam'].astype(np.float32)
    P0 = t.new_tensor(info['calib']['P0'].astype(np.float32))
    cam = _lidar_to_cam(t, rect @ Trv2c)
    corners_img = _points_cam2img(_cam_corners(cam), P0)
    box_2d = torch.cat([torch.min(corners_img, dim=1)[0], torch.max(corners_img, dim=1)[0]],
                       dim=1)
    limit_range = t.new_tensor(pcd_limit_range)
    center = t[:, :3]
    valid = ((center > limit_range[:3]) & (center < limit_range[3:])).all(-1)
    if valid.sum() > 0:
        return dict(bbox=box_2d[valid, :].numpy(), box3d_camera=cam[valid].numpy(),
                    box3d_lidar=t[valid].numpy(), scores=scores[valid].numpy(),
                    label_preds=labels[valid].numpy(), sample_idx=sample_idx)
    return empty


def bbox2result_kitti(results, data_infos, class_names, submission_prefix=None,
                      pcd_limit_range=WAYMO_PCD_LIMIT_RANGE):
    if len(results) != len(data_infos):
        raise ValueError('invalid list length of network outputs')
    if submission_prefix is not None:
        os.makedirs(submission_prefix, exist_ok=True)
    det_annos = []
    for pred_dicts, info in zip(results, data_infos):
        sample_idx = info['image']['image_idx']
        image_shape = info['image']['image_shape'][:2]
        box_dict = convert_valid_bboxes(pred_dicts, info, pcd_limit_range)
        if len(box_dict['bbox']) > 0:
            anno = {k: [] for k in ('name', 'truncated', 'occluded', 'alpha', 'bbox',
                                    'dimensions', 'location', 'rotation_y', 'score')}
            for box, box_lidar, bbox, score, label in zip(
                    box_dict['box3d_camera'], box_dict['box3d_lidar'], box_dict['bbox'],
                    box_dict['scores'], box_dict['label_preds']):
                bbox[2:] = np.minimum(bbox[2:], image_shape[::-1])
                bbox[:2] = np.maximum(bbox[:2], [0, 0])
                anno['name'].append(class_names[int(label)])
                anno['truncated'].append(0.0)
                anno['occluded'].append(0)
                anno['alpha'].append(-np.arctan2(-box_lidar[1], box_lidar[0]) + box[6])
                anno['bbox'].append(bbox)
                anno['dimensions'].append(box[3:6])
                anno['location'].append(box[:3])
                anno['rotation_y'].append(box[6])
                anno['score'].append(score)
            anno = {k: np.stack(v) for k, v in anno.items()}
            if submission_prefix is not None:
                with open(f'{submission_prefix}/{sample_idx:07d}.txt', 'w') as f:
                    bbox, loc, dims = anno['bbox'], anno['location'], anno['dimensions']
                    for i in range(len(bbox)):
                        print('{} -1 -1 {:.4f} {:.4f} {:.4f} {:.4f} '
                              '{:.4f} {:.4f} {:.4f} '
                              '{:.4f} {:.4f} {:.4f} {:.4f} {:.4f} {:.4f}'.format(
                                  anno['name'][i], anno['alpha'][i], bbox[i][0], bbox[i][1],
                                  bbox[i][2], bbox[i][3], dims[i][1], dims[i][2], dims[i][0],
                                  loc[i][0], loc[i][1], loc[i][2], anno['rotation_y'][i],
                                  anno['score'][i]), file=f)
        else:
            anno = {'name': np.array([]), 'truncated': np.array([]), 'occluded': np.array([]),
                    'alpha': np.array([]), 'bbox': np.zeros([0, 4]),
                    'dimensions': np.zeros([0, 3]), 'location': np.zeros([0, 3]),
                    'rotation_y': np.array([]), 'score': np.array([])}
        anno['sample_idx'] = np.array([sample_idx] * len(anno['score']), dtype=np.int64)
        det_annos.append(anno)
    return det_annos
