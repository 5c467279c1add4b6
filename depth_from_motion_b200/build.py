"""In-tree build of the C-ABI CUDA library (nvcc, sm_90a only)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'csrc', 'dfm_b200.cu')
OUT = os.path.join(HERE, 'libdfm_b200.so')
DEPS = [os.path.join(HERE, 'csrc', f) for f in
        ('dfm_b200.cu', 'common.cuh', 'simt_kernels.cuh', 'conv_tc.cuh', 'conv_tc_neck.cuh',
         'neck_api.inc', 'frustum_api.inc', 'frustum_kernels.cuh', 'pipeline_api.inc', 'bev_api.inc', 'tail_kernels.cuh', 'voxel_sample_api.inc', 'stereo_tail_api.inc', 'logits_tc.cuh', 'wgmma.cuh', 'head1x1_tc.cuh', 'anchor3d_head_api.inc', 'spp_neck_kernels.cuh',
         'spp_neck_api.inc', 'fpn_kernels.cuh', 'fpn_api.inc', 'resnet_kernels.cuh',
         'liga_resnet_api.inc', 'resnet101_kernels.cuh', 'resnet101_api.inc',
         'box_post_kernels.cuh', 'box_post_api.inc', 'anchor_loss_kernels.cuh',
         'anchor_loss_api.inc', 'depth_loss_kernels.cuh', 'depth_loss_api.inc',
         'atss_loss_kernels.cuh', 'atss_loss_api.inc', 'imitation_loss_kernels.cuh',
         'imitation_loss_api.inc',
         'image_prep_kernels.cuh',
         'image_prep_api.inc', 'view_cache_kernels.cuh', 'view_cache_api.inc',
         'kitti_eval_kernels.cuh', 'kitti_eval_api.inc', 'waymo_eval_kernels.cuh',
         'waymo_eval_api.inc')] + [os.path.join(HERE, '..', 'include', 'dfm_b200.h')]


def nvcc_path():
    return shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'


def up_to_date():
    if not os.path.isfile(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(d) <= t for d in DEPS)


def build(force=False, verbose=False):
    if up_to_date() and not force:
        return OUT
    cmd = [nvcc_path(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3',
           '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC', '-shared',
           '-o', OUT, SRC]
    if verbose:
        cmd.insert(1, '-Xptxas=-v')
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
