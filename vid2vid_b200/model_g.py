"""Vid2VidModelG on the H100 engine: same public methods and per-clip state as
models/vid2vid_model_G.py (initialize / encode_input / inference / generate_frame_infer /
generate_first_frame / compute_mask / build_pyr), with every tensor op routed to libv2v_b200.so.

Inference only in this round (the reference's own `inference` runs under torch.no_grad,
vid2vid_model_G.py:199); the training forward needs the backward kernels (DESIGN.md, next rows).
"""
import os

import torch
import torch.nn as nn

from .base_model import HostScheduleMixin
from . import networks, ops


def _adam(params, **kw):
    """torch.optim.Adam as the reference builds it; on CUDA parameters the fused multi-tensor implementation (same arithmetic,
    a few dozen launches for ~1000 parameter tensors instead of several hundred)."""
    params = list(params)
    if params and all(p.is_cuda for p in params):
        try:
            return torch.optim.Adam(params, fused=True, **kw)
        except (TypeError, RuntimeError):
            pass
    return torch.optim.Adam(params, **kw)


class Vid2VidModelG(HostScheduleMixin, nn.Module):
    def name(self):
        return 'Vid2VidModelG'

    def initialize(self, opt):
        """vid2vid_model_G.py:19-53 (inference branch)."""
        self.opt = opt
        self.gpu_ids = opt.gpu_ids
        self.isTrain = opt.isTrain
        self.n_scales = opt.n_scales_spatial
        self.use_single_G = opt.use_single_G
        if getattr(opt, 'openpose_only', False):
            opt.no_flow = True
        dev = torch.device('cuda', self.gpu_ids[0] if len(self.gpu_ids) else torch.cuda.current_device())
        self.device_ = dev
        for s in range(self.n_scales):
            setattr(self, 'netG' + str(s), networks.build_netG(opt, s).to(dev))
        # the finest scale reads encode_input's one-hot + edge map at full resolution: exact in bf16 (coarser pyramid levels
        # are avg-pooled, pose inputs are real-valued: not exact)
        getattr(self, 'netG' + str(self.n_scales - 1)).input_exact_bf16 = bool(opt.label_nc != 0)
        # vid2vid_model_G.py:46-51: checkpoints are loaded whenever not training (or continuing / pre-training); a missing G0
        # is an error there (base_model.py:63-72).  opt.synthetic_weights (benchmarks / tests, no checkpoints offline) skips it.
        if (not self.isTrain or getattr(opt, 'continue_train', False) or getattr(opt, 'load_pretrain', '')) and \
                not getattr(opt, 'synthetic_weights', False):
            for s in range(self.n_scales):
                self.load_network(getattr(self, 'netG' + str(s)), 'G' + str(s), opt.which_epoch, getattr(opt, 'load_pretrain', ''))
        self.netG_i = self.load_single_G() if self.use_single_G else None
        self.fake_B_prev = None
        if self.isTrain:
            self.init_train()
        return self

    def load_network(self, network, network_label, epoch_label, save_dir=''):
        """BaseModel.load_network (base_model.py:56-107): <checkpoints_dir>/<name>/<epoch>_net_<label>.pth; a missing G0
        raises, other missing files are reported; on a key / shape mismatch the matching subset is loaded."""
        save_filename = '%s_net_%s.pth' % (epoch_label, network_label)
        save_dir = save_dir or os.path.join(self.opt.checkpoints_dir, self.opt.name)
        save_path = os.path.join(save_dir, save_filename)
        if not os.path.isfile(save_path):
            print('%s not exists yet!' % save_path)
            if 'G0' in network_label:
                raise FileNotFoundError('Generator must exist! (%s)' % save_path)
            return
        sd = torch.load(save_path, map_location=self.device_)
        try:
            network.load_state_dict(sd)
        except Exception:
            own = network.state_dict()
            kept = {k: v for k, v in sd.items() if k in own and v.size() == own[k].size()}
            missing = sorted({k.split('.')[0] for k in own if k not in kept})
            print('Pretrained network %s: loaded %d of %d tensors; not initialised from the file: %s' % (
                network_label, len(kept), len(own), missing))
            own.update(kept)
            network.load_state_dict(own)

    # ------------------------------------------------------------------ first-frame generator
    def load_single_G(self):
        """vid2vid_model_G.py:261-288.  The architecture per dataset / loadSize is the reference's; weights are loaded from
        checkpoints/label2city_single/ or checkpoints/edge2face_single/ (a missing file raises FileNotFoundError naming it, as
        torch.load does in the reference) unless opt.synthetic_weights is set and the file is absent (synthetic benchmarking
        has no checkpoints: seeded initialisation, and for the face model a seeded synthetic features table).  Nothing is
        downloaded."""
        opt = self.opt
        if 'City' in opt.dataroot:
            single_path = 'checkpoints/label2city_single/'
            if opt.loadSize == 512:
                load_path, netG = single_path + 'latest_net_G_512.pth', networks.define_G(35, 3, 0, 64, 'global', 3, 'instance', 0, [], opt)
            elif opt.loadSize == 1024:
                load_path, netG = single_path + 'latest_net_G_1024.pth', networks.define_G(35, 3, 0, 64, 'global', 4, 'instance', 0, [], opt)
            elif opt.loadSize == 2048:
                load_path, netG = single_path + 'latest_net_G_2048.pth', networks.define_G(35, 3, 0, 32, 'local', 4, 'instance', 0, [], opt)
            else:
                raise ValueError('Single image generator does not exist')
        elif 'face' in opt.dataroot:
            single_path = 'checkpoints/edge2face_single/'
            load_path = single_path + 'latest_net_G.pth'
            opt.feat_num = 16
            netG = networks.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], opt)
            self.netE = self._load(networks.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []), single_path + 'latest_net_E.pth')
            self.load_face_features(single_path + 'features.npy')
        else:
            raise ValueError('Single image generator does not exist')
        return self._load(netG, load_path)

    def _load(self, net, path):
        if not (getattr(self.opt, 'synthetic_weights', False) and not os.path.exists(path)):
            if not os.path.exists(path):
                raise FileNotFoundError('first-frame generator weights not found: %s' % path)
            net.load_state_dict(torch.load(path, map_location=self.device_))
        return net.to(self.device_)

    def load_face_features(self, path='checkpoints/edge2face_single/features.npy', features=None):
        """The nearest-neighbour table of get_face_features: `features` ({label: (rows, feat_num + 1)}) if given, else the
        pickled dict at `path` -- read only from that local file, with np.load(encoding='latin1', allow_pickle=True), as the
        reference reads it (vid2vid_model_G.py:295-296) -- else, with opt.synthetic_weights,
        networks.synthetic_face_features(16 rows); otherwise FileNotFoundError naming the path.  Packed once onto the
        device."""
        if features is None:
            if os.path.exists(path):
                import numpy as np
                features = np.load(path, encoding='latin1', allow_pickle=True).item()
            elif getattr(self.opt, 'synthetic_weights', False):
                features = networks.synthetic_face_features(16, self.opt.feat_num, seed=0)
            else:
                raise FileNotFoundError('face features table not found: %s' % path)
        table, self.face_rows, self.face_num_images = networks.pack_face_features(features, self.opt.feat_num)
        self.face_table = table.to(self.device_)
        return features

    # ------------------------------------------------------------------ tensor helpers (CUDA kernels)
    def encode_input(self, input_map, real_image, inst_map=None):
        """vid2vid_model_G.py:86-112."""
        size = input_map.size()
        self.bs, tG, self.height, self.width = size[0], size[1], size[3], size[4]
        input_map = input_map.to(self.device_, torch.float32)
        if self.opt.label_nc != 0:
            inst = inst_map.to(self.device_, torch.float32) if self.opt.use_instance else None
            input_map = ops.onehot_edges(input_map, inst, self.opt.label_nc, self.opt.use_instance)
        elif self.opt.use_instance:
            raise NotImplementedError('use_instance without label_nc')
        pool_map = None
        if self.opt.dataset_mode == 'face':
            pool_map = inst_map.to(self.device_, torch.float32)
        if real_image is not None:
            real_image = real_image.to(self.device_, torch.float32)
        return input_map, real_image, pool_map

    def build_pyr(self, tensor):
        """base_model.py:122-134."""
        if tensor is None:
            return [None] * self.n_scales
        pyr = [tensor]
        for _ in range(1, self.n_scales):
            pyr.append(ops.avgpool3s2(pyr[-1]))
        return pyr

    def compute_mask(self, real_As, ts, te=None):
        """vid2vid_model_G.py:322-330 (single frame)."""
        assert te is None or te == ts + 1
        return ops.fg_mask(real_As, ts, list(self.opt.fg_labels))

    # ------------------------------------------------------------------ inference
    def inference(self, input_A, input_B, inst_A):
        """vid2vid_model_G.py:198-209."""
        with torch.no_grad():
            real_A, real_B, pool_map = self.encode_input(input_A, input_B, inst_A)
            self.is_first_frame = self.fake_B_prev is None
            if self.is_first_frame:
                self.fake_B_prev = self.generate_first_frame(real_A, real_B, pool_map)
            real_A = self.build_pyr(real_A)
            self.fake_B_feat = self.flow_feat = self.fake_B_fg_feat = None
            for s in range(self.n_scales):
                fake_B = self.generate_frame_infer(real_A[self.n_scales - 1 - s], s)
        return fake_B, real_A[0][0, -1]

    # ------------------------------------------------------------------ streaming inference (one new frame per call)
    _DT = {torch.uint8: 0, torch.int32: 1, torch.float32: 2}

    def inference_stream(self, label_frame, inst_frame=None, out_u8=None):
        """Same computation as inference() for a clip fed frame by frame: `label_frame` / `inst_frame` are the NEWEST
        (H, W) id maps (uint8, int32 or float32; host -- ideally pinned -- or device).  The tG-frame id window that
        test.py:31-41 re-sends every step stays resident on the device, so a step uploads one frame.  The first tG - 1
        calls only fill the window and return None.  Returns the generated frame (1, 3, H, W) float, or, when `out_u8`
        (a (H, W, 3) uint8 tensor, host or device) is given, util.tensor2im's uint8 image written into it
        (computed on the device; util/util.py:48-71 does it on the CPU after copying the float frame back)."""
        import ctypes as C
        from . import _lib as L
        if self.opt.dataset_mode == 'face' and self.use_single_G:
            raise ValueError('inference_stream does not take the real frames that the face first-frame generator needs '
                             '(use_single_G with dataset_mode face): use inference()')
        tG = self.opt.n_frames_G
        H, W = label_frame.shape[-2:]
        dev = self.device_
        if getattr(self, '_win_A', None) is None or self._win_A.shape[-2:] != (H, W):
            self._win_A = torch.zeros(1, tG, 1, H, W, device=dev)
            self._win_I = torch.zeros(1, tG, 1, H, W, device=dev) if self.opt.use_instance else None
            self._win_n = 0
        for win, fr in ((self._win_A, label_frame), (self._win_I, inst_frame if inst_frame is not None else label_frame)):
            if win is None:
                continue
            fr = fr.to(dev, non_blocking=True).contiguous()
            if fr.dtype not in self._DT:
                raise TypeError('id maps must be uint8, int32 or float32')
            L.check(L.lib().v2v_ids_window_push(C.c_void_p(win.data_ptr()), C.c_void_p(fr.data_ptr()), self._DT[fr.dtype], tG, H, W,
                                                L.current_stream_ptr()))
            L.LAUNCHES[0] += 1
        self._win_n += 1
        if self._win_n < tG:
            return None
        fake_B, _ = self.inference(self._win_A, None, self._win_I)
        if out_u8 is None:
            return fake_B
        if getattr(self, '_u8_dev', None) is None or self._u8_dev.shape[:2] != (H, W):
            self._u8_dev = torch.empty(H, W, fake_B.shape[1], dtype=torch.uint8, device=dev)
        L.check(L.lib().v2v_tensor2im_u8(C.c_void_p(fake_B.data_ptr()), C.c_void_p(self._u8_dev.data_ptr()), fake_B.shape[1], H, W,
                                         L.current_stream_ptr()))
        L.LAUNCHES[0] += 1
        if out_u8.is_cuda:
            out_u8.copy_(self._u8_dev)
        else:
            out_u8.copy_(self._u8_dev, non_blocking=True)
        return out_u8

    def generate_frame_infer(self, real_A, s):
        """vid2vid_model_G.py:211-229."""
        tG = self.opt.n_frames_G
        _, _, _, h, w = real_A.size()
        si = self.n_scales - 1 - s
        netG_s = getattr(self, 'netG' + str(s))
        real_As_reshaped = real_A[0, :tG].reshape(1, -1, h, w)
        fake_B_prevs_reshaped = self.fake_B_prev[si].reshape(1, -1, h, w)
        mask_F = self.compute_mask(real_A, tG - 1)[0] if self.opt.fg else None
        use_raw_only = self.opt.no_first_img and self.is_first_frame
        fake_B, flow, weight, fake_B_raw, self.fake_B_feat, self.flow_feat, self.fake_B_fg_feat = netG_s.forward(
            real_As_reshaped, fake_B_prevs_reshaped, mask_F, self.fake_B_feat, self.flow_feat, self.fake_B_fg_feat,
            use_raw_only)
        self.fake_B_prev[si] = torch.cat([self.fake_B_prev[si][1:, ...], fake_B])
        return fake_B

    def generate_first_frame(self, real_A, real_B, pool_map=None):
        """vid2vid_model_G.py:231-251."""
        tG = self.opt.n_frames_G
        if self.opt.no_first_img:
            fake_B_prev = torch.zeros(self.bs, tG - 1, self.opt.output_nc, self.height, self.width, device=self.device_)
        elif self.opt.isTrain or self.opt.use_real_img:
            fake_B_prev = real_B[:, :(tG - 1), ...]
        elif self.opt.use_single_G:
            if self.opt.use_instance:
                real_A = real_A[:, :, :self.opt.label_nc, :, :]
            frames = []
            for i in range(tG - 1):
                feat_map = self.get_face_features(real_B[:, i], pool_map[:, i]) if self.opt.dataset_mode == 'face' else None
                frames.append(self.netG_i.forward(real_A[:, i].contiguous(), feat_map).unsqueeze(1))
            fake_B_prev = torch.cat(frames, dim=1)
        else:
            raise ValueError('Please specify the method for generating the first frame')
        fake_B_prev = self.build_pyr(fake_B_prev)
        if not self.opt.isTrain:
            fake_B_prev = [B[0] for B in fake_B_prev]
        return fake_B_prev

    def get_face_features(self, real_image, inst):
        """vid2vid_model_G.py:290-320: the Encoder's pooled features, then the nearest row of the features table (over the
        labels present in `inst`; absent labels do not count, where the reference reads uninitialised memory for them)
        painted over the part map.  One chosen index per call, from the first occurrence of each label over the whole batch.
        self.face_chosen keeps the (1,) int32 device tensor of the index."""
        feat = self.netE.forward(real_image.contiguous(), inst.contiguous())
        feat_map, self.face_chosen = ops.face_features(feat, inst.contiguous(), self.face_table, self.face_rows, self.face_num_images)
        return feat_map

    # ------------------------------------------------------------------ training forward
    def init_train(self):
        """The training half of vid2vid_model_G.py:19-84: per-GPU frame budget and the generator optimizer."""
        opt = self.opt
        self.n_gpus = 1                                                    # one process per GPU (vid2vid_model_G.py:57-61 with n_gpus_gen = 1)
        self.n_frames_per_gpu = min(getattr(opt, 'max_frames_per_gpu', 1), opt.n_frames_total - opt.n_frames_G + 1)
        self.n_frames_load = self.n_gpus * self.n_frames_per_gpu
        self.n_frames_bp = min(getattr(opt, 'max_frames_backpropagate', 1), self.n_frames_load)
        self.finetune_all = True                                           # niter_fix_global == 0 (:66-68)
        params = []
        for s in range(self.n_scales):
            params += list(getattr(self, 'netG' + str(s)).parameters())
        beta1, beta2, lr = (0, 0.9, opt.lr / 2) if opt.TTUR else (opt.beta1, 0.999, opt.lr)       # :74-83
        self.old_lr = opt.lr
        self.optimizer_G = _adam(params, lr=lr, betas=(beta1, beta2))
        return self

    def forward(self, input_A, input_B, inst_A, fake_B_prev, dummy_bs=0):
        """vid2vid_model_G.py:114-140 (one process per GPU: no dummy padding, no frame pipeline over GPUs)."""
        tG = self.opt.n_frames_G
        real_A_all, real_B_all, _ = self.encode_input(input_A, input_B, inst_A)
        is_first_frame = fake_B_prev is None
        if is_first_frame:
            fake_B_prev = self.generate_first_frame(real_A_all, real_B_all)
        fake_B, fake_B_raw, flow, weight = self.generate_frame_train(real_A_all, fake_B_prev, is_first_frame)
        fake_B_prev = [B[:, -tG + 1:].detach() for B in fake_B]
        fake_B = [B[:, tG - 1:] for B in fake_B]
        return fake_B[0], fake_B_raw, flow, weight, real_A_all[:, tG - 1:], real_B_all[:, tG - 2:], fake_B_prev

    def generate_frame_train(self, real_A_all, fake_B_pyr, is_first_frame):
        """vid2vid_model_G.py:142-196."""
        tG, n_scales = self.opt.n_frames_G, self.n_scales
        if not hasattr(self, 'n_frames_load'):
            self.init_train()
        bs = real_A_all.shape[0]
        real_A_pyr = self.build_pyr(real_A_all)
        fake_B_pyr = list(fake_B_pyr)
        fake_Bs_raw, flows, weights = None, None, None
        cat = lambda a, b: b if a is None else torch.cat([a, b], dim=1)
        for t in range(self.n_frames_load):
            fake_B_feat = flow_feat = fake_B_fg_feat = None
            for s in range(n_scales):
                si = n_scales - 1 - s
                real_As = real_A_pyr[si]
                h, w = real_As.shape[-2:]
                real_As_reshaped = real_As[:, t:t + tG].reshape(bs, -1, h, w)
                fake_B_prevs = fake_B_pyr[si][:, t:t + tG - 1]
                if (t % self.n_frames_bp) == 0:
                    fake_B_prevs = fake_B_prevs.detach()
                fake_B_prevs_reshaped = fake_B_prevs.reshape(bs, -1, h, w)
                mask_F = self.compute_mask(real_As, t + tG - 1) if self.opt.fg else None
                use_raw_only = self.opt.no_first_img and is_first_frame
                fake_B, flow, weight, fake_B_raw, fake_B_feat, flow_feat, fake_B_fg_feat = getattr(self, 'netG' + str(s)).forward(
                    real_As_reshaped, fake_B_prevs_reshaped, mask_F, fake_B_feat, flow_feat, fake_B_fg_feat, use_raw_only)
                if s != n_scales - 1 and not self.finetune_all:
                    fake_B, fake_B_feat = fake_B.detach(), fake_B_feat.detach()
                    if flow is not None:
                        flow, flow_feat = flow.detach(), flow_feat.detach()
                    if fake_B_fg_feat is not None:
                        fake_B_fg_feat = fake_B_fg_feat.detach()
                fake_B_pyr[si] = cat(fake_B_pyr[si], fake_B.unsqueeze(1))
                if s == n_scales - 1:
                    fake_Bs_raw = cat(fake_Bs_raw, fake_B_raw.unsqueeze(1))
                    if flow is not None:
                        flows, weights = cat(flows, flow.unsqueeze(1)), cat(weights, weight.unsqueeze(1))
        return fake_B_pyr, fake_Bs_raw, flows, weights

    def save(self, label):
        """vid2vid_model_G.py:338-340."""
        for s in range(self.n_scales):
            self.save_network(getattr(self, 'netG' + str(s)), 'G' + str(s), label, self.gpu_ids)

    def compute_fake_B_prev(self, real_B_prev, fake_B_last, fake_B):
        """vid2vid_model_G.py:332-336."""
        fake_B_prev = real_B_prev[:, 0:1] if fake_B_last is None else fake_B_last[0][:, -1:]
        if fake_B.size()[1] > 1:
            fake_B_prev = torch.cat([fake_B_prev, fake_B[:, :-1].detach()], dim=1)
        return fake_B_prev
