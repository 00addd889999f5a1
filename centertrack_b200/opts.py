"""The subset of the reference's flag system (opts.py:9-403) that the inference hot path reads, with
the same flag names, defaults and derived fields (`parse` 257-326, `update_dataset_info_and_set_heads`
329-388, `init` 390-403).  Training / logging / visualisation flags are accepted and ignored so that
reference command lines keep working.  Extra flag: --b200_precision {bf16,fp32}."""
import argparse

from .dataset_info import dataset_factory


class opts(object):

  def __init__(self):
    p = argparse.ArgumentParser()
    a = p.add_argument
    a('task', default='')
    a('--dataset', default='coco')
    a('--test_dataset', default='')
    a('--debug', type=int, default=0)
    a('--no_pause', action='store_true')
    a('--demo', default='')
    a('--load_model', default='')
    a('--gpus', default='0')
    a('--seed', type=int, default=317)
    a('--arch', default='dla_34')
    a('--dla_node', default='dcn')
    a('--backbone', default='dla34')           # --arch generic (generic_network.py:13-22)
    a('--neck', default='dlaup')
    a('--msra_outchannel', type=int, default=256)
    a('--head_conv', type=int, default=-1)
    a('--num_head_conv', type=int, default=1)
    a('--head_kernel', type=int, default=3)
    a('--down_ratio', type=int, default=4)
    a('--num_classes', type=int, default=-1)
    a('--prior_bias', type=float, default=-4.6)
    a('--input_res', type=int, default=-1)
    a('--input_h', type=int, default=-1)
    a('--input_w', type=int, default=-1)
    a('--ltrb', action='store_true')
    a('--ltrb_weight', type=float, default=0.1)
    a('--reset_hm', action='store_true')
    a('--reuse_hm', action='store_true')
    a('--flip_test', action='store_true')
    a('--test_scales', type=str, default='1')
    a('--K', type=int, default=100)
    a('--fix_short', type=int, default=-1)
    a('--keep_res', action='store_true')
    a('--out_thresh', type=float, default=-1)
    a('--depth_scale', type=float, default=1)
    a('--model_output_list', action='store_true')
    a('--non_block_test', action='store_true')
    a('--test_focal_length', type=int, default=-1)
    a('--tracking', action='store_true')
    a('--pre_hm', action='store_true')
    a('--zero_pre_hm', action='store_true')
    a('--pre_thresh', type=float, default=-1)
    a('--track_thresh', type=float, default=0.3)
    a('--new_thresh', type=float, default=0.3)
    a('--ltrb_amodal', action='store_true')
    a('--ltrb_amodal_weight', type=float, default=0.1)
    a('--public_det', action='store_true')
    a('--no_pre_img', action='store_true')
    a('--zero_tracking', action='store_true')
    a('--hungarian', action='store_true')
    a('--max_age', type=int, default=-1)
    a('--nuscenes_att', action='store_true')
    a('--velocity', action='store_true')
    a('--vis_thresh', type=float, default=0.3)
    a('--save_video', action='store_true')
    a('--resume', action='store_true')
    a('--lr', type=float, default=1.25e-4)
    a('--lr_step', type=str, default='60')
    # loss weights: a head whose weight is 0 is not built (opts.py:366-369), so they shape the network
    for flag, default in (('hm_weight', 1), ('off_weight', 1), ('wh_weight', 0.1), ('hp_weight', 1),
                          ('hm_hp_weight', 1), ('amodel_offset_weight', 1), ('dep_weight', 1), ('dim_weight', 1),
                          ('rot_weight', 1), ('tracking_weight', 1), ('nuscenes_att_weight', 1),
                          ('velocity_weight', 1)):
      a('--' + flag, type=float, default=default)
    a('--b200_precision', default='bf16', choices=['bf16', 'fp32', 'bf16x3'])
    a('--b200_device_pre', action='store_true', help='Detector.run: warpAffine + normalise on the GPU (SURVEY 8f-2)')
    self.parser = p

  def parse(self, args=''):
    opt, ignored = self.parser.parse_known_args() if args == '' else self.parser.parse_known_args(args)
    if ignored:     # training / logging / visualisation flags of the reference are accepted; say so, a typo must be visible
      print('centertrack_b200.opts: ignoring arguments outside the inference path: %s' % ' '.join(ignored))
    opt.ignored_args = ignored
    if opt.test_dataset == '':
      opt.test_dataset = opt.dataset
    opt.gpus_str = opt.gpus
    opt.gpus = [int(g) for g in opt.gpus.split(',')]
    opt.gpus = [i for i in range(len(opt.gpus))] if opt.gpus[0] >= 0 else [-1]
    opt.lr_step = [int(i) for i in opt.lr_step.split(',')]
    opt.test_scales = [float(i) for i in opt.test_scales.split(',')]
    opt.pre_img = False
    # the thresholds as given, before the derivation below: a StreamRunner stream's own flags are derived from them
    opt.thresh_args = {'out_thresh': opt.out_thresh, 'pre_thresh': opt.pre_thresh, 'new_thresh': opt.new_thresh}
    if 'tracking' in opt.task:
      opt.tracking = True
      opt.out_thresh = max(opt.track_thresh, opt.out_thresh)
      opt.pre_thresh = max(opt.track_thresh, opt.pre_thresh)
      opt.new_thresh = max(opt.track_thresh, opt.new_thresh)
      opt.pre_img = not opt.no_pre_img
    opt.fix_res = not opt.keep_res
    if opt.head_conv == -1:
      opt.head_conv = 256 if 'dla' in opt.arch else 64
    opt.pad = 127 if 'hourglass' in opt.arch else 31
    opt.num_stacks = 2 if opt.arch == 'hourglass' else 1
    return opt

  def update_dataset_info_and_set_heads(self, opt, dataset):
    """opts.py:322-388 of the reference: resolution defaults from the dataset, then the head table
    {name: channels} in the reference's insertion order (the state-dict and the decode roles depend on it)."""
    if opt.num_classes < 0:
      opt.num_classes = dataset.num_categories
    default_h, default_w = (opt.input_res, opt.input_res) if opt.input_res > 0 else dataset.default_resolution
    if opt.input_h <= 0:
      opt.input_h = default_h
    if opt.input_w <= 0:
      opt.input_w = default_w
    opt.output_h, opt.output_w = opt.input_h // opt.down_ratio, opt.input_w // opt.down_ratio
    opt.input_res, opt.output_res = max(opt.input_h, opt.input_w), max(opt.output_h, opt.output_w)
    joints = getattr(dataset, 'num_joints', 0)
    head_table = [(True, (('hm', opt.num_classes), ('reg', 2), ('wh', 2))),
                  ('tracking' in opt.task, (('tracking', 2),)),
                  ('ddd' in opt.task, (('dep', 1), ('rot', 8), ('dim', 3), ('amodel_offset', 2))),
                  ('multi_pose' in opt.task, (('hps', 2 * joints), ('hm_hp', joints), ('hp_offset', 2))),
                  (opt.ltrb, (('ltrb', 4),)), (opt.ltrb_amodal, (('ltrb_amodal', 4),)),
                  (opt.nuscenes_att, (('nuscenes_att', 8),)), (opt.velocity, (('velocity', 3),))]
    opt.heads = {name: ch for enabled, group in head_table if enabled for name, ch in group}
    weight_of = {'hm': opt.hm_weight, 'wh': opt.wh_weight, 'reg': opt.off_weight, 'hps': opt.hp_weight,
                 'hm_hp': opt.hm_hp_weight, 'hp_offset': opt.off_weight, 'dep': opt.dep_weight, 'rot': opt.rot_weight,
                 'dim': opt.dim_weight, 'amodel_offset': opt.amodel_offset_weight, 'ltrb': opt.ltrb_weight,
                 'tracking': opt.tracking_weight, 'ltrb_amodal': opt.ltrb_amodal_weight,
                 'nuscenes_att': opt.nuscenes_att_weight, 'velocity': opt.velocity_weight}
    opt.weights = {name: weight_of[name] for name in opt.heads}
    opt.heads = {name: ch for name, ch in opt.heads.items() if opt.weights[name] != 0}   # opts.py:366-369
    width = opt.head_conv
    opt.head_conv = {name: [width] * (1 if name == 'reg' else opt.num_head_conv) for name in opt.heads}
    return opt

  def init(self, args=''):
    default_dataset_info = {
        'ctdet': 'coco', 'multi_pose': 'coco_hp', 'ddd': 'nuscenes', 'tracking,ctdet': 'coco',
        'tracking,multi_pose': 'coco_hp', 'tracking,ddd': 'nuscenes'}
    opt = self.parse(args)
    name = default_dataset_info[opt.task] if opt.task in default_dataset_info else 'coco'
    opt = self.update_dataset_info_and_set_heads(opt, dataset_factory[name])
    return opt
