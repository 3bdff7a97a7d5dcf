"""Vid2VidModelG on the H100 engine: same public methods and per-clip state as
models/vid2vid_model_G.py (initialize / encode_input / inference / generate_frame_infer /
generate_first_frame / compute_mask / build_pyr), with every tensor op routed to libv2v_b200.so.

Inference only in this round (the reference's own `inference` runs under torch.no_grad,
vid2vid_model_G.py:199); the training forward needs the backward kernels (DESIGN.md, next rows).
"""
import collections
import contextlib
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
        for s, net in enumerate(networks.build_netGs(opt)):
            setattr(self, 'netG' + str(s), net.to(dev))
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
        # pretrained and never trained here: with grad mode on, the first frames still run the inference plans
        return net.requires_grad_(False).to(self.device_)

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
        if self.opt.dataset_mode == 'face' and inst_map is not None:
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
        """vid2vid_model_G.py:198-209.  input_A (b, T, C, H, W) holds b independent clips (the reference runs b = 1): the
        generators then run per-sample-statistics plans (_Planned.sample_stats), so every clip's frames equal its own b = 1
        run bit for bit.  The clips of one sequence start and advance together; b == 1 keeps the reference's batch-less
        fake_B_prev."""
        with torch.no_grad():
            real_A, real_B, pool_map = self.encode_input(input_A, input_B, inst_A)
            with self._per_clip_statistics(self.bs > 1):
                return self._inference(real_A, real_B, pool_map)

    @contextlib.contextmanager
    def _per_clip_statistics(self, on):
        """The generators' per-sample-statistics plans (b independent clips, each normalised with its own statistics) for the
        duration of one inference call: afterwards the modules build batch-statistics (and training) plans as before."""
        nets = [getattr(self, 'netG' + str(s)) for s in range(self.n_scales)] + [
            net for net in (self.netG_i, getattr(self, 'netE', None)) if net is not None]
        prev = [getattr(net, 'sample_stats', False) for net in nets]
        for net in nets:
            net.sample_stats = on
        try:
            yield
        finally:
            for net, p in zip(nets, prev):
                net.sample_stats = p

    def _inference(self, real_A, real_B, pool_map):
        self.is_first_frame = self.fake_B_prev is None
        if self.is_first_frame:
            self.fake_B_prev = self.generate_first_frame(real_A, real_B, pool_map)
        elif self.bs != self._clips():
            raise ValueError('this sequence was started with %d clip(s) and is fed %d: clips of one sequence start and advance '
                             'together (reset_stream() starts a new one)' % (self._clips(), self.bs))
        real_A = self.build_pyr(real_A)
        self.fake_B_feat = self.flow_feat = self.fake_B_fg_feat = None
        for s in range(self.n_scales):
            fake_B = self.generate_frame_infer(real_A[self.n_scales - 1 - s], s)
        return fake_B, (real_A[0][0, -1] if self.bs == 1 else real_A[0][:, -1])

    def _clips(self):
        """Clips of the running sequence: fake_B_prev keeps a batch axis only for b > 1 (the reference's b = 1 state has none)."""
        return self.fake_B_prev[0].shape[0] if self.fake_B_prev[0].dim() == 5 else 1

    def reset_stream(self, clips=None):
        """Start a new sequence: the next inference() / inference_stream() call generates first frames again.  `clips` (a
        list of clip indices) asks to restart only some clips of a running batch, which is not supported: the clips of a
        batch start and advance together."""
        n = self._clips() if self.fake_B_prev is not None else 0
        if clips is not None and n > 1 and sorted(set(clips)) != list(range(n)):
            raise NotImplementedError('restarting clip(s) %s of a running batch of %d clips is not supported: the clips of a batch '
                                      'start and advance together; call reset_stream() to restart the whole batch, or use '
                                      'stream_slots(B), whose slots start and stop independently' % (list(clips), n))
        self.fake_B_prev = None
        self._win_A = self._win_I = self._win_B = self._win_P = None

    # ------------------------------------------------------------------ streaming inference (one new frame per call)
    _DT = {torch.uint8: 0, torch.int32: 1, torch.float32: 2}

    def inference_stream(self, label_frame, inst_frame=None, out_u8=None, real_frame=None):
        """Same computation as inference() for a clip fed frame by frame: `label_frame` / `inst_frame` are the NEWEST
        (H, W) id maps (uint8, int32 or float32; host -- ideally pinned -- or device).  The tG-frame id window that
        test.py:31-41 re-sends every step stays resident on the device, so a step uploads one frame.  The first tG - 1
        calls only fill the window and return None.  Returns the generated frame (1, 3, H, W) float, or, when `out_u8`
        (a (H, W, 3) uint8 tensor, host or device) is given, util.tensor2im's uint8 image written into it
        (computed on the device; util/util.py:48-71 does it on the CPU after copying the float frame back).
        B clips at once: (B, H, W) id maps, frames (B, 3, H, W), out_u8 (B, H, W, 3); every step is one launch per helper
        for all clips, and every call of one stream must feed the same B.

        With label_nc 0 (the pose and face demos) `label_frame` is the newest dense frame, (input_nc, H, W) or
        (B, input_nc, H, W) float32, pushed into a resident (B, tG, input_nc, H, W) window.  Face streams (dataset_mode face
        with use_single_G) also take, on each of the first tG - 1 calls, the real frame `real_frame` ((B,) 3, H, W) and the
        part map `inst_frame` ((B,) H, W ids): the first frames are generated from them as inference() generates them from
        real_B[:, :tG - 1] and the part maps; later calls ignore both."""
        import ctypes as C
        from . import _lib as L
        opt, tG, dev = self.opt, self.opt.n_frames_G, self.device_
        B, H, W, batched, fresh = self._stream_frames(label_frame, inst_frame, real_frame)
        face = opt.dataset_mode == 'face' and self.use_single_G
        if fresh:
            self._win_A = torch.zeros(B, tG, opt.input_nc if opt.label_nc == 0 else 1, H, W, device=dev)
            self._win_I = torch.zeros(B, tG, 1, H, W, device=dev) if opt.use_instance else None
            self._win_B = torch.zeros(B, tG - 1, 3, H, W, device=dev) if face else None
            self._win_P = torch.zeros(B, tG - 1, 1, H, W, device=dev) if face else None
            self._win_n = 0
        if opt.label_nc == 0:
            fr = label_frame.to(dev, non_blocking=True).contiguous()
            push = (C.c_int * B)(*[L.SLOT_PUSH] * B)
            L.check(L.lib().v2v_slots_window_push(C.c_void_p(self._win_A.data_ptr()), C.c_void_p(fr.data_ptr()), self._DT[fr.dtype], B,
                                                  tG, opt.input_nc, H, W, push, L.current_stream_ptr()))
            L.LAUNCHES[0] += 1
        else:
            for win, fr in ((self._win_A, label_frame), (self._win_I, inst_frame if inst_frame is not None else label_frame)):
                if win is None:
                    continue
                fr = fr.to(dev, non_blocking=True).contiguous()
                if fr.dtype not in self._DT:
                    raise TypeError('id maps must be uint8, int32 or float32')
                L.check(L.lib().v2v_ids_window_push(C.c_void_p(win.data_ptr()), C.c_void_p(fr.data_ptr()), self._DT[fr.dtype], B, tG,
                                                    H, W, L.current_stream_ptr()))
                L.LAUNCHES[0] += 1
        if face and self._win_n < tG - 1:            # the frames generate_first_frame reads
            self._win_B[:, self._win_n].copy_(real_frame.reshape(B, 3, H, W), non_blocking=True)
            self._win_P[:, self._win_n, 0].copy_(inst_frame.reshape(B, H, W), non_blocking=True)
        self._win_n += 1
        if self._win_n < tG:
            return None
        fake_B, _ = self.inference(self._win_A, self._win_B, self._win_P if face else self._win_I)
        if out_u8 is None:
            return fake_B
        shape = (B, H, W, fake_B.shape[1]) if batched else (H, W, fake_B.shape[1])
        if getattr(self, '_u8_dev', None) is None or tuple(self._u8_dev.shape) != shape:
            self._u8_dev = torch.empty(shape, dtype=torch.uint8, device=dev)
        L.check(L.lib().v2v_tensor2im_u8(C.c_void_p(fake_B.data_ptr()), C.c_void_p(self._u8_dev.data_ptr()), B, fake_B.shape[1], H,
                                         W, L.current_stream_ptr()))
        L.LAUNCHES[0] += 1
        if out_u8.is_cuda:
            out_u8.copy_(self._u8_dev)
        else:
            out_u8.copy_(self._u8_dev, non_blocking=True)
        return out_u8

    def _stream_frames(self, label_frame, inst_frame, real_frame):
        """Checks one inference_stream call's frames against the options and the running stream before anything is
        launched.  Returns (B, H, W, batched: the frames carry a clip axis, fresh: this call starts a new window)."""
        opt, tG = self.opt, self.opt.n_frames_G
        face = opt.dataset_mode == 'face' and self.use_single_G
        win = getattr(self, '_win_A', None)

        def need_face_frames():
            missing = [n for n, t in (('real_frame', real_frame), ('inst_frame (the part map)', inst_frame)) if t is None]
            if missing:
                raise ValueError('a face stream (dataset_mode face with use_single_G) needs %s on each of its first %d calls: the '
                                 'face first-frame generator reads them' % (' and '.join(missing), tG - 1))
        if face and (win is None or self._win_n < tG - 1):
            need_face_frames()
        if opt.label_nc == 0:
            C_ = opt.input_nc
            if label_frame.dim() not in (3, 4) or label_frame.shape[-3] != C_ or label_frame.dtype != torch.float32:
                raise ValueError('label_frame must be a dense (%d, H, W) or (B, %d, H, W) float32 frame (label_nc 0, input_nc %d), '
                                 'got %s %s' % (C_, C_, C_, tuple(label_frame.shape), label_frame.dtype))
            batched = label_frame.dim() == 4
        else:
            batched = label_frame.dim() == 3
            if inst_frame is not None and tuple(inst_frame.shape) != tuple(label_frame.shape):
                raise ValueError('inst_frame %s does not match label_frame %s' % (tuple(inst_frame.shape), tuple(label_frame.shape)))
        B = label_frame.shape[0] if batched else 1
        H, W = label_frame.shape[-2:]
        if win is not None and win.shape[0] != B:
            raise ValueError('this stream was started with %d clip(s) and is fed %d: clips of one stream start and advance '
                             'together (reset_stream() starts a new one)' % (win.shape[0], B))
        fresh = win is None or tuple(win.shape[-2:]) != (H, W)
        if not face:
            if real_frame is not None:
                raise ValueError('real_frame is taken by face streams only (dataset_mode face with use_single_G)')
        elif fresh or self._win_n < tG - 1:
            need_face_frames()                      # a new frame size starts a new window
            lead = (B,) if batched else ()
            for name, t, want in (('real_frame', real_frame, lead + (3, H, W)), ('inst_frame', inst_frame, lead + (H, W))):
                if tuple(t.shape) != want:
                    raise ValueError('%s %s does not match label_frame %s: expected %s' % (
                        name, tuple(t.shape), tuple(label_frame.shape), want))
            if not real_frame.is_floating_point() or inst_frame.dtype not in self._DT:
                raise TypeError('real_frame must be floating point and inst_frame uint8, int32 or float32')
        return B, H, W, batched, fresh

    def stream_slots(self, B):
        """A slot stream (SlotStream) of B slots over this model's generators: every slot starts, restarts and stops its own
        clips, and each clip's frames equal its own batch-1 inference_stream / inference run bit for bit.  Its state is its
        own: this model's inference / inference_stream state is left as it is."""
        return SlotStream(self, B)

    def generate_frame_infer(self, real_A, s):
        """vid2vid_model_G.py:211-229."""
        tG = self.opt.n_frames_G
        b, _, _, h, w = real_A.size()
        si = self.n_scales - 1 - s
        netG_s = getattr(self, 'netG' + str(s))
        real_As_reshaped = real_A[:, :tG].reshape(b, -1, h, w)
        fake_B_prevs_reshaped = self.fake_B_prev[si].reshape(b, -1, h, w)
        mask_F = None
        if self.opt.fg:
            mask_F = self.compute_mask(real_A, tG - 1)
            mask_F = mask_F[0] if b == 1 else mask_F
        use_raw_only = self.opt.no_first_img and self.is_first_frame
        fake_B, flow, weight, fake_B_raw, self.fake_B_feat, self.flow_feat, self.fake_B_fg_feat = netG_s.forward(
            real_As_reshaped, fake_B_prevs_reshaped, mask_F, self.fake_B_feat, self.flow_feat, self.fake_B_fg_feat,
            use_raw_only)
        if b == 1:
            self.fake_B_prev[si] = torch.cat([self.fake_B_prev[si][1:, ...], fake_B])
        else:
            self.fake_B_prev[si] = torch.cat([self.fake_B_prev[si][:, 1:], fake_B.unsqueeze(1)], dim=1)
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
            if self.opt.dataset_mode == 'face' and self.bs == 1:
                for i in range(tG - 1):
                    frames.append(self.netG_i.forward(real_A[:, i].contiguous(), self.get_face_features(
                        real_B[:, i], pool_map[:, i])).unsqueeze(1))
            elif self.opt.dataset_mode == 'face':
                # b independent clips: batch-b per-sample plans (every conv configured as at batch 1) and one table row per
                # clip, so each clip's first frames equal its own b = 1 run bit for bit
                with self._per_clip_statistics(True):
                    for i in range(tG - 1):
                        frames.append(self.netG_i.forward(real_A[:, i].contiguous(), self.get_face_features_per_clip(
                            real_B[:, i], pool_map[:, i])).unsqueeze(1))
            else:
                for i in range(tG - 1):
                    frames.append(self.netG_i.forward(real_A[:, i].contiguous(), None).unsqueeze(1))
            fake_B_prev = torch.cat(frames, dim=1)
        else:
            raise ValueError('Please specify the method for generating the first frame')
        fake_B_prev = self.build_pyr(fake_B_prev)
        if not self.opt.isTrain and self.bs == 1:
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

    def get_face_features_per_clip(self, real_image, inst):
        """get_face_features for b independent clips, one image each: the Encoder runs once on the batch and every image gets
        the nearest table row of its own labels (ops.face_features per_image).  self.face_chosen keeps the (b,) int32 device
        tensor of the indices."""
        feat = self.netE.forward(real_image.contiguous(), inst.contiguous())
        feat_map, self.face_chosen = ops.face_features(feat, inst.contiguous(), self.face_table, self.face_rows, self.face_num_images,
                                                       per_image=True)
        return feat_map

    # ------------------------------------------------------------------ training forward
    def init_train(self):
        """The training half of vid2vid_model_G.py:19-84: per-GPU frame budget and the generator optimizer."""
        opt = self.opt
        self.n_gpus = 1                                                    # one process per GPU (vid2vid_model_G.py:57-61 with n_gpus_gen = 1)
        self.n_frames_per_gpu = min(getattr(opt, 'max_frames_per_gpu', 1), opt.n_frames_total - opt.n_frames_G + 1)
        self.n_frames_load = self.n_gpus * self.n_frames_per_gpu
        self.n_frames_bp = 1                                               # :58; update_training_batch raises it
        # :66-72: with --niter_fix_global only the finest scale trains until update_fixed_params
        self.finetune_all = getattr(opt, 'niter_fix_global', 0) == 0
        scales = range(self.n_scales) if self.finetune_all else [self.n_scales - 1]
        params = [p for s in scales for p in getattr(self, 'netG' + str(s)).parameters()]
        beta1, beta2, lr = (0.0, 0.9, opt.lr / 2) if opt.TTUR else (opt.beta1, 0.999, opt.lr)       # :74-83
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
                # :181-186 detaches a frozen coarser scale's outputs; running it without autograd gives the same values from
                # the inference plan (batch statistics and the running-statistics update included), with no saved
                # statistics and no gradient buffers
                frozen = s != n_scales - 1 and not self.finetune_all
                with torch.no_grad() if frozen else contextlib.nullcontext():
                    fake_B, flow, weight, fake_B_raw, fake_B_feat, flow_feat, fake_B_fg_feat = getattr(self, 'netG' + str(s)).forward(
                        real_As_reshaped, fake_B_prevs_reshaped, mask_F, fake_B_feat, flow_feat, fake_B_fg_feat, use_raw_only)
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


class SlotStep(collections.namedtuple('SlotStep', 'ops ready join raw_only')):
    """What one SlotStream step does per slot: the window op (v2v_slots_window_push, _lib.SLOT_*), whether the slot produces
    a frame (ready), whether this is its clip's first produced frame (join: its previous frames are seeded first) and
    whether that frame takes the raw composite (raw_only: a join under --no_first_img)."""

    def flags(self):
        """The per-image flags of the generators' slot plans (_lib.IMAGE_ACTIVE | IMAGE_RAW_ONLY)."""
        from . import _lib as L
        return [(L.IMAGE_ACTIVE if r else 0) | (L.IMAGE_RAW_ONLY if o else 0) for r, o in zip(self.ready, self.raw_only)]


class SlotSchedule:
    """Host bookkeeping of a slot stream: B slots, each feeding its clip through a tG-frame window.  start(k) (a new clip,
    restarting a busy slot) and stop(k) (the slot goes idle) take effect at the next step().  A slot produces a frame once its
    window holds tG frames of its clip, so a clip's first tG - 1 steps produce nothing, as with inference_stream."""

    def __init__(self, B, tG, no_first_img=False):
        from . import _lib as L
        if not 1 <= B <= L.MAX_SLOTS:
            raise ValueError('a slot stream has 1 to %d slots, not %d' % (L.MAX_SLOTS, B))
        self.B, self.tG, self.no_first_img = B, tG, bool(no_first_img)
        self.frames = [0] * B          # frames of the slot's running clip so far (0: idle)
        self._next = [None] * B        # 'start' / 'stop' at the next step

    def _slot(self, k):
        if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k < self.B:
            raise IndexError('slot %r is out of range for a stream of %d slots' % (k, self.B))
        return k

    def start(self, k):
        self._next[self._slot(k)] = 'start'

    def stop(self, k):
        self._next[self._slot(k)] = 'stop'

    def step(self):
        from . import _lib as L
        ops = []
        for k in range(self.B):
            nxt, self._next[k] = self._next[k], None
            if nxt == 'start':
                self.frames[k] = 1
                ops.append(L.SLOT_RESTART)
            elif nxt == 'stop':
                self.frames[k] = 0
                ops.append(L.SLOT_CLEAR)
            elif self.frames[k]:
                self.frames[k] += 1
                ops.append(L.SLOT_PUSH)
            else:
                ops.append(L.SLOT_KEEP)
        ready = [n >= self.tG for n in self.frames]
        join = [n == self.tG for n in self.frames]
        return SlotStep(ops, ready, join, [j and self.no_first_img for j in join])


class SlotStream:
    """B slots over one set of per-sample generator plans (Vid2VidModelG.stream_slots).  Every slot starts a clip, restarts
    with a new one or goes idle between steps; the batch shape never changes, so each scale keeps one slot plan and one CUDA
    graph.  Slots that are idle or still filling their window are computed but produce nothing and leave the running
    statistics alone: every clip's frames, and the running statistics, are those of its own batch-1 run."""

    def __init__(self, model, B):
        opt = model.opt
        if opt.dataset_mode == 'face' and model.use_single_G:
            raise ValueError('a slot stream does not take the real frames that the face first-frame generator needs '
                             '(use_single_G with dataset_mode face): use inference()')
        if not (opt.no_first_img or (model.use_single_G and not opt.use_real_img)):
            raise ValueError('a slot stream seeds the first frames of a joining clip with --no_first_img or --use_single_G '
                             '(it takes no real frames)')
        self.model, self.B, self.tG = model, B, opt.n_frames_G
        self.schedule = SlotSchedule(B, self.tG, opt.no_first_img)
        self.C = 1 if opt.label_nc != 0 else opt.input_nc
        self._win_A = self._win_I = self.fake_B_prev = self._flags = self._u8_dev = None

    def start(self, k):
        """Slot k begins a new clip at its next frame (restarting it if busy)."""
        self.schedule.start(k)

    def stop(self, k):
        """Slot k goes idle from its next step on."""
        self.schedule.stop(k)

    def _check(self, frames, inst):
        B, opt = self.B, self.model.opt
        if opt.label_nc != 0:
            if frames.dim() != 3 or frames.shape[0] != B:
                raise ValueError('frames must be (%d, H, W) id maps, got %s' % (B, tuple(frames.shape)))
            if frames.dtype not in Vid2VidModelG._DT:
                raise TypeError('id maps must be uint8, int32 or float32')
        elif frames.dim() != 4 or tuple(frames.shape[:2]) != (B, self.C) or frames.dtype != torch.float32:
            raise ValueError('frames must be (%d, %d, H, W) float32, got %s %s' % (B, self.C, tuple(frames.shape), frames.dtype))
        if inst is not None and (tuple(inst.shape) != tuple(frames.shape) or inst.dtype not in Vid2VidModelG._DT):
            raise ValueError('inst %s does not match frames %s' % (tuple(inst.shape), tuple(frames.shape)))
        H, W = frames.shape[-2:]
        if self._win_A is not None and tuple(self._win_A.shape[-2:]) != (H, W):
            raise ValueError('this slot stream runs %dx%d frames, got %dx%d' % (self._win_A.shape[-2], self._win_A.shape[-1], H, W))
        return H, W

    def step(self, frames, inst=None, out_u8=None):
        """One frame for every slot: `frames` are the slots' newest frames, (B, H, W) id maps (uint8 / int32 / float32) when
        label_nc != 0 or (B, input_nc, H, W) float32 frames, host or device; rows of idle slots are ignored.  Returns
        (frames, ready): the generated (B, 3, H, W) float frames -- or `out_u8` ((B, H, W, 3) uint8, host or device) filled
        with util.tensor2im's images -- and a host list of B bools, ready[k] = slot k produced a frame this step."""
        import ctypes as C
        from . import _lib as L
        m, opt, B, tG = self.model, self.model.opt, self.B, self.tG
        H, W = self._check(frames, inst)
        dev = m.device_
        if self._win_A is None:
            self._win_A = torch.zeros(B, tG, self.C, H, W, device=dev)
            self._win_I = torch.zeros(B, tG, 1, H, W, device=dev) if opt.use_instance else None
            self.fake_B_prev, h, w = [], H, W
            for _ in range(m.n_scales):            # build_pyr's level extents
                self.fake_B_prev.append(torch.zeros(B, tG - 1, opt.output_nc, h, w, device=dev))
                h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            self._flags = torch.zeros(B, dtype=torch.int32, device=dev)
        st = self.schedule.step()
        ops = (C.c_int * B)(*st.ops)
        for win, fr in ((self._win_A, frames), (self._win_I, inst if inst is not None else frames)):
            if win is None:
                continue
            fr = fr.to(dev, non_blocking=True).contiguous()
            L.check(L.lib().v2v_slots_window_push(C.c_void_p(win.data_ptr()), C.c_void_p(fr.data_ptr()), Vid2VidModelG._DT[fr.dtype],
                                                  B, tG, win.shape[2], H, W, ops, L.current_stream_ptr()))
            L.LAUNCHES[0] += 1
        # one asynchronous pinned copy: the slot plans read the flags through their IO tables, so their graphs stay valid
        self._flags.copy_(torch.tensor(st.flags(), dtype=torch.int32).pin_memory(), non_blocking=True)
        with torch.no_grad():
            real_A, _, _ = m.encode_input(self._win_A, None, self._win_I)
            for k in range(B):
                if st.join[k]:
                    self._seed_first_frames(real_A, k)
            real_A = m.build_pyr(real_A)
            feats = (None, None, None)
            with m._per_clip_statistics(True):
                for s in range(m.n_scales):
                    si = m.n_scales - 1 - s
                    ra = real_A[si]
                    h, w = ra.shape[-2:]
                    mask = m.compute_mask(ra, tG - 1) if opt.fg else None
                    fake_B, _, _, _, *feats = getattr(m, 'netG' + str(s)).forward(
                        ra[:, :tG].reshape(B, -1, h, w), self.fake_B_prev[si].reshape(B, -1, h, w), mask, *feats, False,
                        image_flags=self._flags)
                    self.fake_B_prev[si] = torch.cat([self.fake_B_prev[si][:, 1:], fake_B.unsqueeze(1)], dim=1)
        if out_u8 is None:
            return fake_B, st.ready
        if self._u8_dev is None or tuple(self._u8_dev.shape) != (B, H, W, fake_B.shape[1]):
            self._u8_dev = torch.empty(B, H, W, fake_B.shape[1], dtype=torch.uint8, device=dev)
        L.check(L.lib().v2v_tensor2im_u8(C.c_void_p(fake_B.data_ptr()), C.c_void_p(self._u8_dev.data_ptr()), B, fake_B.shape[1], H,
                                         W, L.current_stream_ptr()))
        L.LAUNCHES[0] += 1
        out_u8.copy_(self._u8_dev, non_blocking=not out_u8.is_cuda)
        return out_u8, st.ready

    def _seed_first_frames(self, real_A, k):
        """Slot k's previous frames when its window first fills: zeros (--no_first_img, with the raw composite this step) or
        netG_i on the first tG - 1 frames of its window at batch 1 (--use_single_G), as generate_first_frame makes them for
        a batch-1 run, copied into the slot's rows of every scale."""
        m, opt = self.model, self.model.opt
        if opt.no_first_img:
            for prev in self.fake_B_prev:
                prev[k].zero_()
            return
        a = real_A[k:k + 1, :, :opt.label_nc] if opt.use_instance else real_A[k:k + 1]
        first = torch.cat([m.netG_i.forward(a[:, i].contiguous(), None).unsqueeze(1) for i in range(self.tG - 1)], dim=1)
        for prev, p in zip(self.fake_B_prev, m.build_pyr(first)):
            prev[k] = p[0]
