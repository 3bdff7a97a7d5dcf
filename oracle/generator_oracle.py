"""TEST INFRASTRUCTURE -- not product code.  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / `--impl reference` leg may import this.

CPU restatement (PyTorch functional ops, fp32) of the reference's per-frame hot path:
generators, discriminator towers, warp / composite, pyramid, one-hot + edges, and the
`Vid2VidModelG.inference()` driver.  Every function cites the reference lines it follows.
Parameters come from a state_dict with the reference's own key names, so the same
dict drives the reference modules (oracle/ref_shim.py), this restatement and the CUDA path.

Parity pin: there are no reference tests / golden vectors (SURVEY.md 4) -> the pin is the
reference itself: oracle/make_golden.py runs the reference modules on seeded inputs and stores their
outputs in tests/golden/, and tests/test_oracle_vs_reference.py / tests/test_oracle_vs_golden.py check
every function here against them (bit-exact or <=1e-5).
"""
import torch
import torch.nn.functional as F

EPS = 1e-5


# ----------------------------------------------------------------------------- layers
def _norm(x, sd, p, kind):
    """get_norm_layer (models/networks.py:23-30).  Both norms run in *training* mode at
    inference (SURVEY App. B #1): batch statistics of the current tensor."""
    if kind == 'batch':
        return F.batch_norm(x, None, None, sd[p + '.weight'], sd[p + '.bias'], True, 0.1, EPS)
    elif kind == 'instance':
        return F.instance_norm(x, None, None, None, None, True, 0.1, EPS)
    raise NotImplementedError(kind)


def _conv(x, sd, p, stride=1, padding=0):
    return F.conv2d(x, sd[p + '.weight'], sd[p + '.bias'], stride=stride, padding=padding)


def _deconv(x, sd, p):
    # nn.ConvTranspose2d(k=3, stride=2, padding=1, output_padding=1)  networks.py:147,176,254,272
    return F.conv_transpose2d(x, sd[p + '.weight'], sd[p + '.bias'], stride=2, padding=1, output_padding=1)


def _stem7(x, sd, p, i, kind, act=True):
    """[ReflectionPad2d(3), Conv7x7, norm, ReLU] at Sequential indices i..i+3 (networks.py:153)."""
    x = _conv(F.pad(x, (3, 3, 3, 3), mode='reflect'), sd, '%s.%d' % (p, i + 1))
    x = _norm(x, sd, '%s.%d' % (p, i + 2), kind)
    return F.relu(x)


def _down(x, sd, p, i, kind):
    """[Conv3x3 s2 p1, norm, ReLU] at indices i..i+2 (networks.py:156-157)."""
    x = _conv(x, sd, '%s.%d' % (p, i), stride=2, padding=1)
    return F.relu(_norm(x, sd, '%s.%d' % (p, i + 1), kind))


def _up(x, sd, p, i, kind):
    """[ConvTranspose3x3 s2, norm, ReLU] at indices i..i+2 (networks.py:176-177)."""
    x = _deconv(x, sd, '%s.%d' % (p, i))
    return F.relu(_norm(x, sd, '%s.%d' % (p, i + 1), kind))


def _resblock(x, sd, p, kind):
    """ResnetBlock.forward (networks.py:591-593); conv_block = [RPad1, Conv3, norm, ReLU,
    RPad1, Conv3, norm] (networks.py:559-589)."""
    h = _conv(F.pad(x, (1, 1, 1, 1), mode='reflect'), sd, p + '.conv_block.1')
    h = F.relu(_norm(h, sd, p + '.conv_block.2', kind))
    h = _conv(F.pad(h, (1, 1, 1, 1), mode='reflect'), sd, p + '.conv_block.5')
    h = _norm(h, sd, p + '.conv_block.6', kind)
    return x + h


def _head7(x, sd, p):
    """[ReflectionPad2d(3), Conv7x7] (+ activation applied by caller) networks.py:178,182,183."""
    return _conv(F.pad(x, (3, 3, 3, 3), mode='reflect'), sd, p + '.1')


# ----------------------------------------------------------------------------- warp
def get_grid(b, rows, cols):
    """get_grid (networks.py:79-93)."""
    hor = torch.linspace(-1.0, 1.0, cols).view(1, 1, 1, cols).expand(b, 1, rows, cols)
    ver = torch.linspace(-1.0, 1.0, rows).view(1, 1, rows, 1).expand(b, 1, rows, cols)
    return torch.cat([hor, ver], 1)


def resample(image, flow, align_corners=False):
    """BaseNetwork.resample / grid_sample (networks.py:102-115).  The reference passes no
    align_corners: PyTorch 0.4 behaved as True, the installed torch defaults to False
    (SURVEY App. B #2) -- the flag is explicit here."""
    b, c, h, w = image.size()
    grid = get_grid(b, h, w)
    flow = torch.cat([flow[:, 0:1] / ((w - 1.0) / 2.0), flow[:, 1:2] / ((h - 1.0) / 2.0)], dim=1)
    final_grid = (grid + flow).permute(0, 2, 3, 1)
    return F.grid_sample(image, final_grid, mode='bilinear', padding_mode='border',
                         align_corners=align_corners)


# ----------------------------------------------------------------------------- generators
def composite_generator(sd, inp, img_prev, mask, use_raw_only=False, *, n_downsampling=3, n_blocks=9,
                        use_fg_model=True, no_flow=False, norm='batch', align_corners=False,
                        flow_multiplier=20.0):
    """CompositeGenerator.forward (networks.py:203-232); layer indices follow the
    constructor (networks.py:128-201)."""
    nd = n_downsampling

    def down_branch(x, p):
        x = _stem7(x, sd, p, 0, norm)
        for i in range(nd):
            x = _down(x, sd, p, 4 + 3 * i, norm)
        for i in range(n_blocks - n_blocks // 2):
            x = _resblock(x, sd, '%s.%d' % (p, 4 + 3 * nd + i), norm)
        return x

    def res_up(x, pres, pup):
        for i in range(n_blocks // 2):
            x = _resblock(x, sd, '%s.%d' % (pres, i), norm)
        for i in range(nd):
            x = _up(x, sd, pup, 3 * i, norm)
        return x

    downsample = down_branch(inp, 'model_down_seg') + down_branch(img_prev, 'model_down_img')   # :204
    img_feat = res_up(downsample, 'model_res_img', 'model_up_img')                                # :205
    img_raw = torch.tanh(_head7(img_feat, sd, 'model_final_img'))                                 # :206
    flow = weight = flow_feat = None
    if not no_flow:
        flow_feat = res_up(downsample, 'model_res_flow', 'model_up_flow')                         # :210-211
        flow = _head7(flow_feat, sd, 'model_final_flow') * flow_multiplier                        # :212
        weight = torch.sigmoid(_head7(flow_feat, sd, 'model_final_w'))                            # :213
    if use_raw_only or no_flow:
        img_final = img_raw
    else:
        img_warp = resample(img_prev[:, -3:], flow, align_corners)                                # :219
        w_ = weight.expand_as(img_raw)
        img_final = img_raw * w_ + img_warp * (1 - w_)                                            # :221
    img_fg_feat = None
    if use_fg_model:
        x = _stem7(inp, sd, 'indv_down', 0, norm)
        for i in range(nd):
            x = _down(x, sd, 'indv_down', 4 + 3 * i, norm)
        for i in range(n_blocks):
            x = _resblock(x, sd, 'indv_res.%d' % i, norm)
        for i in range(nd):
            x = _up(x, sd, 'indv_up', 3 * i, norm)
        img_fg_feat = x                                                                           # :225
        img_fg = torch.tanh(_head7(img_fg_feat, sd, 'indv_final'))                                # :226
        m = mask.expand_as(img_raw)
        img_final = img_fg * m + img_final * (1 - m)                                              # :229
        img_raw = img_fg * m + img_raw * (1 - m)                                                  # :230
    return img_final, flow, weight, img_raw, img_feat, flow_feat, img_fg_feat


def composite_local_generator(sd, inp, img_prev, mask, img_feat_coarse, flow_feat_coarse, img_fg_feat_coarse,
                              use_raw_only=False, *, n_blocks_local=3, use_fg_model=True, no_flow=False,
                              norm='batch', scale=1, align_corners=False):
    """CompositeLocalGenerator.forward (networks.py:296-325); constructor :235-294."""
    flow_multiplier = 20 * (2 ** scale)                                                           # :297

    def down(x, p):
        x = _stem7(x, sd, p, 0, norm)
        return _down(x, sd, p, 4, norm)

    def up(x, p):
        for i in range(n_blocks_local):
            x = _resblock(x, sd, '%s.%d' % (p, i), norm)
        return _up(x, sd, p, n_blocks_local, norm)

    down_img = down(inp, 'model_down_seg') + down(img_prev, 'model_down_img')                     # :298
    img_feat = up(down_img + img_feat_coarse, 'model_up_img')                                     # :299
    img_raw = torch.tanh(_head7(img_feat, sd, 'model_final_img'))
    flow = weight = flow_feat = None
    if not no_flow:
        flow_feat = up(down_img + flow_feat_coarse, 'model_up_flow')                              # :305
        flow = _head7(flow_feat, sd, 'model_final_flow') * flow_multiplier                        # :306
        weight = torch.sigmoid(_head7(flow_feat, sd, 'model_final_w'))
    if use_raw_only or no_flow:
        img_final = img_raw
    else:
        img_warp = resample(img_prev[:, -3:], flow, align_corners)
        w_ = weight.expand_as(img_raw)
        img_final = img_raw * w_ + img_warp * (1 - w_)
    img_fg_feat = None
    if use_fg_model:
        img_fg_feat = up(down(inp, 'indv_down') + img_fg_feat_coarse, 'indv_up')                  # :319
        img_fg = torch.tanh(_head7(img_fg_feat, sd, 'indv_final'))
        m = mask.expand_as(img_raw)
        img_final = img_fg * m + img_final * (1 - m)
        img_raw = img_fg * m + img_raw * (1 - m)
    return img_final, flow, weight, img_raw, img_feat, flow_feat, img_fg_feat


def _global_trunk(x, sd, p, n_downsampling, n_blocks, norm, with_final):
    """GlobalGenerator.model (networks.py:335-353)."""
    x = _stem7(x, sd, p, 0, norm)
    i = 4
    for _ in range(n_downsampling):
        x = _down(x, sd, p, i, norm)
        i += 3
    for _ in range(n_blocks):
        x = _resblock(x, sd, '%s.%d' % (p, i), norm)
        i += 1
    for _ in range(n_downsampling):
        x = _up(x, sd, p, i, norm)
        i += 3
    if with_final:
        x = torch.tanh(_conv(F.pad(x, (3, 3, 3, 3), mode='reflect'), sd, '%s.%d' % (p, i + 1)))
    return x


def global_generator(sd, inp, *, n_downsampling=3, n_blocks=9, norm='instance'):
    """GlobalGenerator.forward (networks.py:355-359)."""
    return _global_trunk(inp, sd, 'model', n_downsampling, n_blocks, norm, True)


def avgpool3s2(x):
    """AvgPool2d(3, stride=2, padding=1, count_include_pad=False) (networks.py:400,652;
    base_model.py:129)."""
    return F.avg_pool2d(x, 3, stride=2, padding=1, count_include_pad=False)


def local_enhancer(sd, inp, *, n_downsample_global=4, n_blocks_global=9, n_local_enhancers=1,
                   n_blocks_local=3, norm='instance'):
    """LocalEnhancer.forward (networks.py:402-419); constructor :362-400."""
    pyr = [inp]
    for _ in range(n_local_enhancers):
        pyr.append(avgpool3s2(pyr[-1]))
    out = _global_trunk(pyr[-1], sd, 'model', n_downsample_global, n_blocks_global, norm, False)
    for n in range(1, n_local_enhancers + 1):
        p1, p2 = 'model%d_1' % n, 'model%d_2' % n
        x = _stem7(pyr[n_local_enhancers - n], sd, p1, 0, norm)
        x = _down(x, sd, p1, 4, norm) + out
        for i in range(n_blocks_local):
            x = _resblock(x, sd, '%s.%d' % (p2, i), norm)
        x = _up(x, sd, p2, n_blocks_local, norm)
        if n == n_local_enhancers:
            x = torch.tanh(_conv(F.pad(x, (3, 3, 3, 3), mode='reflect'), sd, '%s.%d' % (p2, n_blocks_local + 4)))
        out = x
    return out


# ----------------------------------------------------------------------------- discriminator
def multiscale_discriminator(sd, inp, *, num_D=3, n_layers=3, norm='batch', getIntermFeat=True):
    """MultiscaleDiscriminator.forward (networks.py:663-675) over NLayerDiscriminator towers
    (networks.py:685-706): Conv4x4 s2 p2 + LReLU | (n_layers-1) x [Conv4x4 s2 p2, norm, LReLU] |
    Conv4x4 s1 p2, norm, LReLU | Conv4x4 s1 p2."""
    assert getIntermFeat
    result = []
    x = inp
    for i in range(num_D):
        d = num_D - 1 - i
        feats = []
        h = x
        for j in range(n_layers + 2):
            p = 'scale%d_layer%d' % (d, j)
            stride = 2 if j < n_layers else 1
            h = _conv(h, sd, p + '.0', stride=stride, padding=2)
            if 0 < j < n_layers + 1:
                h = _norm(h, sd, p + '.1', norm)
            if j < n_layers + 1:
                h = F.leaky_relu(h, 0.2)
            feats.append(h)
        result.append(feats)
        if i != num_D - 1:
            x = avgpool3s2(x)
    return result


# ----------------------------------------------------------------------------- model_G level
def get_edges(t):
    """BaseModel.get_edges (base_model.py:146-152): 4-neighbour instance-boundary map."""
    edge = torch.zeros(t.size(), dtype=torch.bool)
    edge[..., :, 1:] |= (t[..., :, 1:] != t[..., :, :-1])
    edge[..., :, :-1] |= (t[..., :, 1:] != t[..., :, :-1])
    edge[..., 1:, :] |= (t[..., 1:, :] != t[..., :-1, :])
    edge[..., :-1, :] |= (t[..., 1:, :] != t[..., :-1, :])
    return edge.float()


def encode_input(input_map, inst_map, label_nc, use_instance):
    """Vid2VidModelG.encode_input (vid2vid_model_G.py:86-112): one-hot scatter of label ids +
    instance edge channel.  input_map (b,t,1,H,W) float ids -> (b,t,label_nc[+1],H,W)."""
    b, t, _, h, w = input_map.size()
    if label_nc != 0:
        oh = torch.zeros(b, t, label_nc, h, w)
        oh.scatter_(2, input_map.long(), 1.0)
        input_map = oh
    if use_instance:
        input_map = torch.cat([input_map, get_edges(inst_map)], dim=2)
    return input_map


def build_pyr(tensor, n_scales):
    """BaseModel.build_pyr (base_model.py:122-134)."""
    pyr = [tensor]
    for _ in range(1, n_scales):
        b, t, c, h, w = pyr[-1].size()
        down = avgpool3s2(pyr[-1].view(-1, h, w).unsqueeze(0)).squeeze(0).view(b, t, c, h // 2, w // 2)
        pyr.append(down)
    return pyr


def compute_mask(real_As, ts, fg_labels):
    """Vid2VidModelG.compute_mask (vid2vid_model_G.py:322-330)."""
    m = real_As[:, ts:ts + 1, fg_labels[0]].clone()
    for l in fg_labels[1:]:
        m = m + real_As[:, ts:ts + 1, l]
    return torch.clamp(m, 0, 1)


class ModelGOracle:
    """Stateful restatement of Vid2VidModelG.inference (vid2vid_model_G.py:198-251).
    `sds[s]` = state_dict of netG{s}; `sd_single` = state_dict of the first-frame generator
    (`--use_single_G`, vid2vid_model_G.py:261-276) with `single_kind` in {'global','local'}."""

    def __init__(self, opt, sds, sd_single=None, single_kind='global', single_nd=3, align_corners=False):
        self.opt, self.sds, self.sd_single = opt, sds, sd_single
        self.single_kind, self.single_nd = single_kind, single_nd
        self.align_corners = align_corners
        self.n_scales = opt.n_scales_spatial
        self.fake_B_prev = None

    def _first_frames(self, real_A):
        opt = self.opt
        tG = opt.n_frames_G
        b, _, _, h, w = real_A.size()
        if opt.no_first_img:                                                      # :233-234
            prev = torch.zeros(b, tG - 1, opt.output_nc, h, w)
        elif opt.use_single_G:                                                    # :237-244
            a = real_A[:, :, :opt.label_nc] if opt.use_instance else real_A
            frames = []
            for i in range(tG - 1):
                if self.single_kind == 'global':
                    f = global_generator(self.sd_single, a[:, i], n_downsampling=self.single_nd,
                                         n_blocks=opt.n_blocks, norm='instance')
                else:
                    f = local_enhancer(self.sd_single, a[:, i], n_downsample_global=self.single_nd,
                                       n_blocks_global=opt.n_blocks, n_local_enhancers=opt.n_local_enhancers,
                                       n_blocks_local=opt.n_blocks_local, norm='instance')
                frames.append(f.unsqueeze(1))
            prev = torch.cat(frames, dim=1)
        else:
            raise ValueError('Please specify the method for generating the first frame')
        return [B[0] for B in build_pyr(prev, self.n_scales)]                      # :248-250

    def inference(self, input_A, inst_A):
        opt = self.opt
        tG = opt.n_frames_G
        real_A = encode_input(input_A, inst_A, opt.label_nc, opt.use_instance)   # :200
        is_first = self.fake_B_prev is None
        if is_first:
            self.fake_B_prev = self._first_frames(real_A)                         # :203
        pyr = build_pyr(real_A, self.n_scales)                                    # :205
        feats = (None, None, None)
        fake_B = None
        for s in range(self.n_scales):                                            # :207-208
            si = self.n_scales - 1 - s
            rA = pyr[si]
            _, _, _, h, w = rA.size()
            a = rA[0, :tG].reshape(1, -1, h, w)                                   # :218
            prevs = self.fake_B_prev[si].reshape(1, -1, h, w)                     # :219
            mask = compute_mask(rA, tG - 1, opt.fg_labels)[0] if opt.fg else None  # :220
            raw_only = opt.no_first_img and is_first                             # :221
            if s == 0:
                out = composite_generator(self.sds[0], a, prevs, mask, raw_only,
                                          n_downsampling=opt.n_downsample_G, n_blocks=opt.n_blocks,
                                          use_fg_model=opt.fg, no_flow=opt.no_flow, norm=opt.norm,
                                          align_corners=self.align_corners)
            else:
                out = composite_local_generator(self.sds[s], a, prevs, mask, feats[0], feats[1], feats[2],
                                                raw_only, n_blocks_local=opt.n_blocks_local,
                                                use_fg_model=opt.fg, no_flow=opt.no_flow, norm=opt.norm,
                                                scale=s, align_corners=self.align_corners)
            fake_B = out[0]
            feats = (out[4], out[5], out[6])
            self.fake_B_prev[si] = torch.cat([self.fake_B_prev[si][1:], fake_B])  # :228
        return fake_B, pyr[0][0, -1]

    def _generate(self, s, a, prevs, mask, feats, raw_only):
        opt = self.opt
        if s == 0:
            return composite_generator(self.sds[0], a, prevs, mask, raw_only, n_downsampling=opt.n_downsample_G,
                                       n_blocks=opt.n_blocks, use_fg_model=opt.fg, no_flow=opt.no_flow, norm=opt.norm,
                                       align_corners=self.align_corners)
        return composite_local_generator(self.sds[s], a, prevs, mask, feats[0], feats[1], feats[2], raw_only,
                                         n_blocks_local=opt.n_blocks_local, use_fg_model=opt.fg, no_flow=opt.no_flow,
                                         norm=opt.norm, scale=s, align_corners=self.align_corners)

    def train_forward(self, input_A, input_B, inst_A, fake_B_prev=None, n_frames_load=1):
        """Vid2VidModelG.forward in training (vid2vid_model_G.py:114-140) with generate_frame_train (:142-196) and the
        training branch of generate_first_frame (:231-251), single process (no GPU pipeline, dummy_bs = 0), forward
        values only (detach points do not change them).  input_A / inst_A: (b, n_frames_load + tG - 1, 1, H, W) label
        and instance ids, input_B: the real frames.  Returns the reference's 7-tuple: fake_B (b, n_frames_load, 3, H, W),
        fake_B_raw, flow, weight, real_A[:, tG-1:], real_B[:, tG-2:], fake_B_prev pyramid for the next call."""
        opt = self.opt
        tG = opt.n_frames_G
        real_A = encode_input(input_A, inst_A, opt.label_nc, opt.use_instance)
        b = real_A.size(0)
        first = fake_B_prev is None
        if first:                                                                 # :231-248
            if opt.no_first_img:
                prev = torch.zeros(b, tG - 1, opt.output_nc, real_A.size(3), real_A.size(4))
            else:
                prev = input_B[:, :tG - 1]                                         # training: the first frames are given
            fake_B_prev = build_pyr(prev, self.n_scales)
        pyr_B = [p for p in fake_B_prev]
        pyr_A = build_pyr(real_A, self.n_scales)                                  # :151
        raws, flows, weights = [], [], []
        for t in range(n_frames_load):                                            # :155
            feats = (None, None, None)
            for s in range(self.n_scales):                                        # :161-162
                si = self.n_scales - 1 - s
                rA = pyr_A[si]
                h, w = rA.shape[-2:]
                a = rA[:, t:t + tG].reshape(b, -1, h, w)                          # :167
                prevs = pyr_B[si][:, t:t + tG - 1].reshape(b, -1, h, w)           # :170-173
                mask = compute_mask(rA, t + tG - 1, opt.fg_labels) if opt.fg else None   # :176
                out = self._generate(s, a, prevs, mask, feats, opt.no_first_img and first)
                feats = (out[4], out[5], out[6])
                pyr_B[si] = torch.cat([pyr_B[si], out[0].unsqueeze(1)], dim=1)     # :191
                if s == self.n_scales - 1:                                        # :192-196
                    raws.append(out[3].unsqueeze(1))
                    if out[1] is not None:
                        flows.append(out[1].unsqueeze(1))
                        weights.append(out[2].unsqueeze(1))
        cat = lambda l: torch.cat(l, dim=1) if l else None
        next_prev = [B[:, -tG + 1:] for B in pyr_B]                               # :137
        return (pyr_B[0][:, tG - 1:], cat(raws), cat(flows), cat(weights), real_A[:, tG - 1:], input_B[:, tG - 2:], next_prev)
