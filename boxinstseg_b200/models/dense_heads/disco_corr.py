"""f4: DiscoBox's semantic-correspondence path (mmdet/models/dense_heads/discobox_head.py): the per-class object bank
(``ObjectElements`` / ``ObjectQueues`` :69-226), ``SemanticCorrSolver.solve`` (:369-411) and the per-object body of
``corr_loss`` (:1059-1125: retrieval, solve, InfoNCE term, transfer of the retrieved masks into the query's box, bank update).

The reference runs the body object by object; here ALL objects of a level go through it at once (``corr_level``), with the
same sequential semantics: object i sees the bank exactly as the objects before it -- those of its own level included --
left it.  A fixed number of launches per level, whatever the number of objects, and no host synchronisation:
  * retrieval (:174-221) of every query against the virtual bank of its class: ONE launch of ``bxs_corr_retrieve``;
  * cosine tables ``Cu`` (:386-391) of all (query, retrieved) pairs: gathers + normalise + one batched ``torch.matmul`` (a
    library GEMM, and the only part with a gradient -- to the queries' RoI features);
  * the regularised tables ``T`` (:393-410): ONE launch of ``bxs_corr_solve`` over the level's n x max_retrieval_objs tables
    (the unused ones cost nothing);
  * the InfoNCE terms (:1080-1084): batched, masked per query; the count ``num`` stays on the device;
  * the transfer (:1086-1096 + ``superres_T`` :851-865): ONE launch pair of ``bxs_corr_transfer`` -- none of the reference's
    six [K,784,784] intermediates (12 MB each at K = 5) exists;
  * resizing the two 28 x 28 maps to each query's box and writing them into ``iiu`` (:1098-1107): ``bxs_corr_paste``;
  * the ring append (:1113-1124): ``bxs_corr_bank_append``.
The bank is ONE packed device store per ``ObjectQueues`` (feature / mask / box of every (class, slot), int32 ``ptr`` and
``exists`` per class); the head's "first query" state (:1060-1066) is a device flag too.

Third party and absent from the reference checkout: ``mmcv.ops.RoIAlign`` -- the RoI features / masks are inputs here
(``torchvision.ops.roi_align(x, rois, size, 1.0, 0, True)`` is the same operator).
"""
import torch
import torch.nn.functional as F

from ... import _lib as L


def relu_and_l2_norm_feat(feat, dim=1):
    """:16-20."""
    feat = F.relu(feat)
    norm = ((feat ** 2).sum(dim=dim, keepdim=True) + 1e-6) ** 0.5
    return feat / (norm + 1e-6)


class ObjectElements:
    """:69-130: ``size`` slots of (mask [ms,ms], feature [C,fs,fs], box [4]) of one category."""

    def __init__(self, size=100, img_size=0, feat_size=28, mask_size=56, n_channel=256, device='cpu', category=None):
        self.mask = torch.zeros(size, mask_size, mask_size, device=device)
        self.feature = torch.zeros(size, n_channel, feat_size, feat_size, device=device)
        self.box = torch.zeros(size, 4, device=device)
        self.img = None
        self.category = int(category)
        self.ptr = 0

    def get_category(self):
        return self.category

    def get_feature(self):
        return self.feature

    def get_mask(self):
        return self.mask

    def get_box(self):
        return self.box

    def get_ratio(self):
        b = self.box
        return (b[:, 2] - b[:, 0]) / (b[:, 3] - b[:, 1] + 1e-5)

    def __len__(self):
        return len(self.feature)

    def __getitem__(self, idx):
        if isinstance(idx, int):
            idx = slice(idx, idx + 1)
        elif torch.is_tensor(idx):
            idx = idx.to(self.mask.device).long()
        return dict(img=None, mask=self.mask[idx], feature=self.feature[idx], box=self.box[idx], category=self.category)


def create_one(mask, feature, box, category):
    """ObjectFactory.create_one (:26-44): a one-slot holder of the query; the feature is re-normalised like there."""
    q = ObjectElements(size=1, feat_size=feature.shape[2], mask_size=mask.shape[1], n_channel=feature.shape[1],
                       device=mask.device, category=category)
    q.mask[...] = mask
    q.feature[...] = relu_and_l2_norm_feat(feature[0:1])
    q.box[...] = box
    return q


class _BankView(ObjectElements):
    """Class c of a packed store as an ``ObjectElements``: ``feature`` / ``mask`` / ``box`` are views of the store's rows
    [c*L, (c+1)*L); ``ptr`` reads (synchronises) and writes the store's device pointer."""

    def __init__(self, queues, c):                       # noqa -- no slot allocation: the store owns the memory
        rows = slice(c * queues.len_queue, (c + 1) * queues.len_queue)
        self._queues = queues
        self.feature, self.mask, self.box = queues.feature[rows], queues.mask[rows], queues.box[rows]
        self.img = None
        self.category = int(c)

    @property
    def ptr(self):
        return int(self._queues.ptr[self.category])

    @ptr.setter
    def ptr(self, value):
        self._queues.ptr[self.category] = int(value)


class _BankList:
    """``ObjectQueues.queues``: ``queues[c]`` is None until class c has a bank (a read of the device ``exists`` flag:
    synchronises -- for inspection), else a ``_BankView``; assigning an ``ObjectElements`` loads it into the store, assigning
    None drops the class's bank."""

    def __init__(self, queues):
        self._q = queues

    def __len__(self):
        return self._q.num_class

    def __getitem__(self, c):
        q = self._q
        if not -q.num_class <= c < q.num_class:
            raise IndexError(c)
        c %= q.num_class
        if q.feature is None or not bool(q.exists[c]):
            return None
        return _BankView(q, c)

    def __setitem__(self, c, elems):
        self._q.load(c % self._q.num_class, elems)

    def __iter__(self):
        return (self[c] for c in range(len(self)))


class ObjectQueues:
    """:132-226, same constructor arguments.  ONE packed store for all classes: ``feature`` [num_class*L,C,fh,fw], ``mask``
    [num_class*L,mh,mw], ``box`` [num_class*L,4] (class c owns rows [c*L, (c+1)*L)), int32 ``ptr`` / ``exists``
    [num_class]; allocated (zeros) on the first use, from the feature / mask shapes and the device it sees there.  The
    reference keeps one holder per class and spills to host memory after ``num_gpu_bank`` classes: 80 classes x 100 slots x
    (128 x 7 x 7 + 28 x 28) floats = 226 MB here, all on the device."""

    def __init__(self, num_class, len_queue, fg_iou_thresh, bg_iou_thresh, ratio_range, appear_thresh, max_retrieval_objs):
        self.num_class = num_class
        self.len_queue = len_queue
        self.fg_iou_thresh = fg_iou_thresh
        self.bg_iou_thresh = bg_iou_thresh
        self.appear_thresh = appear_thresh
        self.ratio_range = ratio_range
        self.max_retrieval_objs = max_retrieval_objs
        self.feature = self.mask = self.box = self.ptr = self.exists = None
        self.queues = _BankList(self)

    def allocate(self, n_channel, feat_hw, mask_hw, device):
        """The store for features [n_channel, *feat_hw] and masks [*mask_hw] on ``device`` (zeros); a no-op when it exists
        with these shapes.  No data-dependent step: callable before anything is known about the objects."""
        feat_hw, mask_hw, device = tuple(int(v) for v in feat_hw), tuple(int(v) for v in mask_hw), torch.device(device)
        if self.feature is not None:
            if (self.feature.shape[1:] != (n_channel,) + feat_hw or self.mask.shape[1:] != mask_hw or
                    self.feature.device != device):
                raise ValueError(f'object bank holds {tuple(self.feature.shape[1:])} / {tuple(self.mask.shape[1:])} features / '
                                 f'masks on {self.feature.device}, got {(n_channel,) + feat_hw} / {mask_hw} on {device}')
            return
        rows = self.num_class * self.len_queue
        self.feature = torch.zeros((rows, n_channel) + feat_hw, device=device)
        self.mask = torch.zeros((rows,) + mask_hw, device=device)
        self.box = torch.zeros(rows, 4, device=device)
        self.ptr = torch.zeros(self.num_class, dtype=torch.int32, device=device)
        self.exists = torch.zeros(self.num_class, dtype=torch.int32, device=device)

    @torch.no_grad()
    def load(self, c, elems):
        """Class c's bank := ``elems`` (an ``ObjectElements`` of ``len_queue`` slots, its ``ptr`` included); None drops it."""
        if elems is None:
            if self.exists is not None:
                self.exists[c] = 0
                self.ptr[c] = 0
            return
        if len(elems) != self.len_queue:
            raise ValueError(f'a bank has {self.len_queue} slots, got {len(elems)}')
        self.allocate(elems.feature.shape[1], elems.feature.shape[2:], elems.mask.shape[1:], elems.mask.device)
        rows = slice(c * self.len_queue, (c + 1) * self.len_queue)
        self.feature[rows] = elems.feature
        self.mask[rows] = elems.mask
        self.box[rows] = elems.box
        self.ptr[c] = int(elems.ptr)
        self.exists[c] = 1

    @torch.no_grad()
    def append(self, class_idx, idx, feature, mask, box, img=None, device=None):
        """:146-172: entry ``idx`` of the three batched tensors goes to the class's write pointer.  True when the bank was
        created by this call.  One object at a time, reading the pointer on the host (the batched path is ``corr_level``)."""
        self.allocate(feature.shape[1], feature.shape[2:], mask.shape[1:], device or mask.device)
        created = not bool(self.exists[class_idx])
        p = int(self.ptr[class_idx])
        row = class_idx * self.len_queue + p
        self.feature[row] = feature[idx]
        self.mask[row] = mask[idx]
        self.box[row] = box[idx]
        self.ptr[class_idx] = (p + 1) % self.len_queue
        self.exists[class_idx] = 1
        return created

    @torch.no_grad()
    def similar_indices(self, qobj):
        """The slots of the query's class that pass the four tests of get_similar_obj (:205-221), ascending, at most
        ``max_retrieval_objs`` -- as a device tensor (no synchronisation here), or None without a bank."""
        k = self.queues[qobj.get_category()]
        if k is None:
            return None
        A, B = qobj.get_mask(), k.get_mask().to(qobj.get_mask())
        fg = (A * B).sum([1, 2]) / ((A + B) >= 1).float().sum([1, 2])                                        # :174-180
        bg = ((1 - A) * (1 - B)).sum([1, 2]) / ((2 - A - B) >= 1).float().sum([1, 2])                        # :182-186
        f0, f1 = qobj.get_feature(), k.get_feature().to(qobj.get_feature())
        a = F.interpolate(A[:, None], f0.shape[2:], mode='bilinear', align_corners=False)[:, 0]              # :188-199
        b = F.interpolate(B[:, None], f1.shape[2:], mode='bilinear', align_corners=False)[:, 0]
        appear = (f0 * f1 * a[:, None] * b[:, None]).sum([1, 2, 3]) / ((a * b).sum([1, 2]) + 1e-6)
        ratio = (qobj.get_ratio()[:, None] / k.get_ratio()[None, :].to(A))[0]                                # :201-205
        keep = ((fg > self.fg_iou_thresh) & (bg > self.bg_iou_thresh) & (appear > self.appear_thresh) &
                (ratio >= self.ratio_range[0]) & (ratio <= self.ratio_range[1]))
        return torch.where(keep)[0][:self.max_retrieval_objs]

    def get_similar_obj(self, qobj):
        """:205-226: dict(mask, feature, box, category) of the retrieved slots, or None."""
        idx = self.similar_indices(qobj)
        return None if idx is None else self.queues[qobj.get_category()][idx]


class SemanticCorrSolver:
    """:229-411, same constructor arguments (the optimal-transport and Hough-space helpers of the reference class are dead
    code on this path and are not rebuilt)."""

    def __init__(self, exp, eps, gaussian_filter_size, low_score, num_iter, num_smooth_iter, dist_kernel):
        self.exp = exp
        self.eps = eps
        self.gaussian_filter_size = gaussian_filter_size
        self.low_score = low_score
        self.num_iter = num_iter
        self.num_smooth_iter = num_smooth_iter
        self.dist_kernel = dist_kernel

    def cosine_table(self, f0, f1):
        """:386-391: f0 [1,C,h,w], f1 [K,C,h,w] -> Cu [K,P,P] (differentiable w.r.t. f0)."""
        return self.cosine_tables(f0, f1[None])[0]

    def cosine_tables(self, f0, f1):
        """:386-391 for n queries at once: f0 [n,C,h,w], f1 [n,K,C,h,w] -> Cu [n,K,P,P] (differentiable w.r.t. f0)."""
        a = f0.float().reshape(f0.shape[0], 1, f0.shape[1], -1).transpose(3, 2)                        # [n,1,P,C]
        b = f1.float().reshape(f1.shape[0], f1.shape[1], f1.shape[2], -1)                                # [n,K,C,P]
        a = a / (torch.norm(a, p=2, dim=3, keepdim=True) + 1e-4)
        b = b / (torch.norm(b, p=2, dim=2, keepdim=True) + 1e-4)
        with torch.autocast('cuda', enabled=False):
            return torch.matmul(a, b)

    @torch.no_grad()
    def votes(self, Cu, h, w, counts=None):
        """:393-410: the regularised table for a given Cu [K,P,P] (one launch).  No gradient: the reference uses T only
        through argmax and inside no_grad (:1081,1086-1088).  With ``counts`` (int32 [n], K = n * kmax), table j of query q
        is solved only for j < counts[q]; the others are zeros."""
        Cu = Cu.detach().contiguous().float()
        L.require_cuda(Cu, counts)
        T = torch.empty_like(Cu)
        n = counts.shape[0] if counts is not None else 1
        with torch.cuda.device(Cu.device):
            L.check(L.lib().bxs_corr_solve_batched(L.ptr(Cu), L.ptr(T), L.ptr(counts), n, Cu.shape[0] // n, h, w,
                                                   int(self.dist_kernel), int(self.num_iter), int(self.num_smooth_iter),
                                                   L.stream()), 'corr_solve')
        return T

    def solve(self, qobjs, kobjs, f0, return_masks=False):
        """The reference's signature.  Returns (Cu, C, fg_mask, bg_mask); the two [K,M,M] mask products (:378-379) are only
        built on request -- ``transfer`` does not need them."""
        m0 = qobjs.mask.float()
        f1 = kobjs['feature'].to(m0).float()
        m1 = kobjs['mask'].to(m0).float()
        Cu = self.cosine_table(f0, f1)
        C = self.votes(Cu, f0.shape[2], f0.shape[3])
        if not return_masks:
            return Cu, C, None, None
        fg_mask = m0.reshape(m0.shape[0], -1, 1) * m1.reshape(m1.shape[0], 1, -1)
        bg_mask = (1 - m0).reshape(m0.shape[0], -1, 1) * (1 - m1).reshape(m1.shape[0], 1, -1)
        return Cu, C, fg_mask, bg_mask

    @torch.no_grad()
    def transfer(self, T, Cu, qmask, kmask, h, w):
        """:1086-1096 + superres_T: T, Cu [K,P,P], qmask [1,Hm,Wm], kmask [K,Hm,Wm] -> (fg_ci, bg_ci) [Hm,Wm]."""
        fg, bg = self.transfer_batched(T, Cu, qmask, kmask, h, w)
        return fg[0], bg[0]

    @torch.no_grad()
    def transfer_batched(self, T, Cu, qmask, kmask, h, w, counts=None):
        """The transfer for n queries in one launch pair: T, Cu [n*kmax,P,P], qmask [n,Hm,Wm], kmask [n*kmax,Hm,Wm], counts
        int32 [n] (None: kmax tables each) -> (fg_ci, bg_ci) [n,Hm,Wm], the mean over each query's counts[q] tables (zeros
        for a query without any)."""
        T, Cu = T.contiguous().float(), Cu.detach().contiguous().float()
        m0, m1 = qmask.detach().contiguous().float(), kmask.detach().contiguous().float()
        L.require_cuda(T, Cu, m0, m1, counts)
        n, (K, Hm, Wm) = m0.shape[0], m1.shape
        fg = torch.empty((n, Hm, Wm), dtype=torch.float32, device=T.device)
        bg = torch.empty_like(fg)
        lib = L.lib()
        ws = torch.empty(lib.bxs_corr_transfer_workspace_bytes(K, Hm, Wm), dtype=torch.uint8, device=T.device)
        with torch.cuda.device(T.device):
            L.check(lib.bxs_corr_transfer_batched(L.ptr(T), L.ptr(Cu), L.ptr(m0), L.ptr(m1), L.ptr(counts), L.ptr(fg),
                                                  L.ptr(bg), L.ptr(ws), n, K // n, h, w, Hm, Wm, L.stream()), 'corr_transfer')
        return fg, bg


def corr_level(solver, queues, first, roi_s_feat, roi_t_feat, roi_s_mask, roi_t_mask, boxes, labels, valid, iiu, min_size,
               min_objs=5):
    """The per-object body of ``corr_loss`` (:1056-1125) for ALL n objects of one level, with the reference's sequential
    semantics, on the device and without host synchronisation (a fixed number of launches for any n).

    roi_s_feat [n,C,h,w] (student RoI features, normalised, carries the gradient), roi_t_feat / roi_s_mask / roi_t_mask
    (detached RoI tensors), boxes [n,4] (x1,y1,x2,y2 on the mask-feature grid, integer valued), labels [n], valid [n] bool
    (False: the object takes no part -- an all-zero target), iiu [2n,H,W] zeros, first: the head's int32 [1] device flag
    "no query seen yet" (consumed by the first valid object).  Object i:
      1. retrieves from the bank of its class as the objects before it left it (``bxs_corr_retrieve``);
      2. with >= min_objs retrieved: adds its InfoNCE term, transfers the retrieved masks and pastes them over its box into
         iiu[2i] (background) / iiu[2i+1] (foreground);
      3. appends its teacher RoI feature / mask and box when both box sides exceed min_size (``bxs_corr_bank_append``).
    Returns (sum of the InfoNCE terms, number of terms as a device int32 scalar, the retrieval record: dict of int32 src
    [n,kmax], count, kcount, slot, exists [n] -- see include/boxseg_b200.h, bxs_corr_retrieve)."""
    n, C, h, w = roi_s_feat.shape
    Hm, Wm = roi_s_mask.shape[1:]
    H, W = iiu.shape[1:]
    dev = roi_s_feat.device
    queues.allocate(C, (h, w), (Hm, Wm), dev)
    if n == 0:
        none = torch.empty(0, dtype=torch.int32, device=dev)
        return roi_s_feat.new_zeros(()), none.sum(dtype=torch.int32), dict(src=none.view(0, 1), count=none, kcount=none,
                                                                           slot=none, exists=none)
    kmax = max(int(queues.max_retrieval_objs), 1)
    P = h * w
    qf = roi_s_feat.detach().float().contiguous()
    qf_first = relu_and_l2_norm_feat(qf).contiguous()                   # ObjectFactory.create_one (:43)
    tf = roi_t_feat.detach().float().contiguous()
    sm, tm = roi_s_mask.detach().float().contiguous(), roi_t_mask.detach().float().contiguous()
    bx = boxes.detach().float().contiguous()
    lab, val = labels.to(torch.int32).contiguous(), valid.to(torch.int32).contiguous()
    L.require_cuda(qf, tf, sm, tm, bx, lab, val, iiu, first, queues.feature)
    src = torch.empty((n, kmax), dtype=torch.int32, device=dev)
    count, kcount, slot, exists = torch.empty((4, n), dtype=torch.int32, device=dev).unbind(0)
    lib = L.lib()
    with torch.cuda.device(dev):
        L.check(lib.bxs_corr_retrieve(
            L.ptr(queues.feature), L.ptr(queues.mask), L.ptr(queues.box), L.ptr(queues.ptr), L.ptr(queues.exists), L.ptr(first),
            L.ptr(qf), L.ptr(qf_first), L.ptr(sm), L.ptr(tf), L.ptr(tm), L.ptr(bx), L.ptr(lab), L.ptr(val), L.ptr(src),
            L.ptr(count), L.ptr(kcount), L.ptr(slot), L.ptr(exists), n, queues.num_class, queues.len_queue, C, h, w, Hm, Wm,
            float(queues.fg_iou_thresh), float(queues.bg_iou_thresh), float(queues.appear_thresh),
            float(queues.ratio_range[0]), float(queues.ratio_range[1]), float(min_size), int(queues.max_retrieval_objs),
            int(min_objs), L.stream()), 'corr_retrieve')
    # the retrieved objects: rows of the store, or this level's own appended objects (their teacher RoI tensors)
    own = (src < 0).reshape(-1)
    bank_row = torch.where(own, 0, src.reshape(-1)).long()
    lvl_row = torch.where(own, -1 - src.reshape(-1), 0).long()
    f1 = torch.where(own[:, None], tf.reshape(n, -1).index_select(0, lvl_row),
                     queues.feature.reshape(queues.feature.shape[0], -1).index_select(0, bank_row))
    m1 = torch.where(own[:, None], tm.reshape(n, -1).index_select(0, lvl_row),
                     queues.mask.reshape(queues.mask.shape[0], -1).index_select(0, bank_row))
    Cu = solver.cosine_tables(roi_s_feat, f1.view(n, kmax, C, h, w))                 # [n,kmax,P,P]
    T = solver.votes(Cu.reshape(n * kmax, P, P), h, w, counts=kcount)
    # :1080-1084 -- cross entropy of softmax(Cu) against argmax(T), the mean over the K_i * P rows of each query
    asg = T.view(n, kmax, P, P).argmax(3, keepdim=True)
    ce = -F.log_softmax(F.softmax(Cu.float(), 3), 3).gather(3, asg)[..., 0]        # [n,kmax,P]
    used = torch.arange(kmax, device=dev)[None, :] < kcount[:, None]                 # [n,kmax]
    per_query = torch.where(used[..., None], ce, 0).sum((1, 2)) / (kcount.clamp(min=1) * P)
    loss = per_query.sum()
    num = (kcount > 0).sum(dtype=torch.int32)
    fg, bg = solver.transfer_batched(T, Cu, sm, m1.view(n * kmax, Hm, Wm), h, w, counts=kcount)
    with torch.cuda.device(dev):
        L.check(lib.bxs_corr_paste(L.ptr(fg), L.ptr(bg), L.ptr(bx), L.ptr(kcount), L.ptr(iiu), n, Hm, Wm, H, W, L.stream()),
                'corr_paste')
        L.check(lib.bxs_corr_bank_append(L.ptr(queues.feature), L.ptr(queues.mask), L.ptr(queues.box), L.ptr(queues.ptr),
                                         L.ptr(queues.exists), L.ptr(first), L.ptr(tf), L.ptr(tm), L.ptr(bx), L.ptr(lab),
                                         L.ptr(val), L.ptr(slot), n, queues.num_class, queues.len_queue, C * P, Hm * Wm,
                                         L.stream()), 'corr_bank_append')
    return loss, num, dict(src=src, count=count, kcount=kcount, slot=slot, exists=exists)


def corr_objects(solver, queues, qobj, roi_s_feat, roi_t_feat, roi_s_mask, roi_t_mask, boxes, kernel_labels, iiu,
                 objbank_min_size, min_objs=5):
    """The per-object loop of ``corr_loss`` (:1056-1125) for the n objects of one level, all of them valid: ``corr_level``
    with a host count.

    roi_s_feat [n,C,h,w] (student RoI features, normalised, carries the gradient), roi_t_feat / roi_s_mask / roi_t_mask
    (detached RoI tensors), boxes [n,4] (x1,y1,x2,y2 on the mask-feature grid, integer valued), kernel_labels [n], iiu
    [2n,H,W] zeros.  Returns (sum of the InfoNCE terms, number of terms (a host int: synchronises), qobj); fills ``iiu`` and
    updates the bank.  ``qobj`` is the head's one-slot query holder (None on the first call, :1060-1066)."""
    n = roi_s_feat.shape[0]
    dev = roi_s_feat.device
    first = torch.full((1,), int(qobj is None), dtype=torch.int32, device=dev)
    valid = torch.ones(n, dtype=torch.bool, device=dev)
    loss, num, _ = corr_level(solver, queues, first, roi_s_feat, roi_t_feat, roi_s_mask, roi_t_mask, boxes, kernel_labels,
                              valid, iiu, objbank_min_size, min_objs)
    if qobj is None and n > 0:                                           # the holder of the last query, like the reference's
        qobj = create_one(roi_s_mask[n - 1:].detach(), roi_s_feat[n - 1:].detach(), boxes[n - 1:].detach(),
                          int(kernel_labels[n - 1]))
    return loss, int(num), qobj


def _torchvision_roi_align(out_size):
    """mmcv.ops.RoIAlign(out_size) with its defaults (spatial_scale 1, adaptive sampling, aligned=True) -- third party to the
    reference; torchvision ships the same operator."""
    from torchvision.ops import roi_align

    def run(x, rois):
        return roi_align(x, rois, out_size, 1.0, 0, True)
    return run


def mask_boxes(target):
    """The tight box of every non-empty target mask, (min_x, min_y, max_x + 1, max_y + 1) as float (:1029-1035, where the
    reference loops over the objects with four ``.min()/.max()`` host reads each): four reductions, no synchronisation."""
    n, H, W = target.shape
    on = target > 0
    rows, cols = on.any(2), on.any(1)                                        # [n,H], [n,W]
    ys = torch.arange(H, device=target.device)
    xs = torch.arange(W, device=target.device)
    min_y = torch.where(rows, ys, ys.new_full((), H)).amin(1)
    max_y = torch.where(rows, ys, ys.new_full((), -1)).amax(1) + 1
    min_x = torch.where(cols, xs, xs.new_full((), W)).amin(1)
    max_x = torch.where(cols, xs, xs.new_full((), -1)).amax(1) + 1
    return torch.stack([min_x, min_y, max_x, max_y], 1).float()


class DiscoCorr:
    """The state and the per-level body of ``DiscoBoxSOLOv2Head.corr_loss`` (:900-1139) after the dynamic convolutions: per
    level, box every target, RoI-align the student / teacher features and masks, run the per-object body for all objects at
    once (``corr_level``), then the mean field WITH the transferred inter-image maps and the dice against its pseudo labels.
    Objects with an all-zero target (which the reference drops, :1024-1028) stay in the level with a placeholder box and take
    no part in anything.  Built from the head's ``loss_corr`` config dict (:720-749)."""

    def __init__(self, num_classes, loss_corr, roi_align=_torchvision_roi_align):
        bank = loss_corr['obj_bank']
        self.solver = SemanticCorrSolver(loss_corr['corr_exp'], loss_corr['corr_eps'], loss_corr['gaussian_filter_size'],
                                         loss_corr['low_score'], loss_corr['corr_num_iter'], loss_corr['corr_num_smooth_iter'],
                                         dist_kernel=loss_corr['dist_kernel'])
        self.object_queues = ObjectQueues(num_class=num_classes, len_queue=bank['len_object_queues'],
                                          fg_iou_thresh=bank['fg_iou_thresh'], bg_iou_thresh=bank['bg_iou_thresh'],
                                          ratio_range=bank['ratio_range'], appear_thresh=bank['appear_thresh'],
                                          max_retrieval_objs=bank['max_retrieval_objs'])
        self.feat_roi_align = roi_align((bank['feat_height'], bank['feat_width']))
        self.mask_roi_align = roi_align((bank['mask_height'], bank['mask_width']))
        self.feat_hw = (bank['feat_height'], bank['feat_width'])
        self.mask_hw = (bank['mask_height'], bank['mask_width'])
        self.objbank_min_size = bank['min_size']
        self.min_objs = 5                                                    # the literal of :1075
        self.corr_loss_weight = loss_corr['loss_weight']
        self.first = None              # int32 [1] on the device: no query seen yet (the reference's ``qobj is None``)
        self._qobj = None

    @property
    def qobj(self):
        """The reference's query holder: None until the first query (reads the device flag: synchronises; inspection only)."""
        first = self._qobj is None if self.first is None else bool(self.first.item())
        return None if first else (self._qobj if self._qobj is not None else True)

    @qobj.setter
    def qobj(self, value):
        self._qobj = value
        if self.first is not None:
            self.first.fill_(int(value is None))

    def _state(self, s_feat):
        """The bank store and the first-query flag on s_feat's device (allocated on the first call: run one call eagerly
        before capturing this in a CUDA graph)."""
        self.object_queues.allocate(s_feat.shape[1], self.feat_hw, self.mask_hw, s_feat.device)
        if self.first is None:
            self.first = torch.full((1,), int(self._qobj is None), dtype=torch.int32, device=s_feat.device)

    def levels_masked(self, s_ins_pred_list, t_ins_pred_list, img_ind_list, ins_labels, kernel_label_list, s_feat, t_feat,
                      mean_field, use_ind_teacher=False):
        """``levels`` without host synchronisation: returns (corr_loss / (num + 1e-4), [(dice terms [n_l], valid [n_l] bool)
        per level with objects]); the terms of objects with an all-zero target are 0 and not valid."""
        self._state(s_feat)
        total = s_feat.new_zeros(())
        num = torch.zeros((), dtype=torch.int32, device=s_feat.device)
        out = []
        for s_in, t_in, img_inds, target, klabels in zip(s_ins_pred_list, t_ins_pred_list, img_ind_list, ins_labels,
                                                         kernel_label_list):
            if s_in is None or s_in.shape[0] == 0:
                continue
            valid = (target.flatten(1) != 0).any(1)                           # the reference drops the others (:1024-1028)
            s = torch.sigmoid(s_in)
            t = torch.sigmoid(t_in) if use_ind_teacher else s
            img_inds = img_inds.to(s.device)
            n = s.shape[0]
            placeholder = (torch.arange(4, device=s.device) >= 2).float()     # (0, 0, 1, 1): RoIAlign of an empty target
            boxes = torch.where(valid[:, None], mask_boxes(target), placeholder)
            rois = torch.cat([img_inds.to(s_feat)[:, None], boxes], 1)
            roi_s_feat = relu_and_l2_norm_feat(self.feat_roi_align(s_feat, rois))
            with torch.no_grad():
                roi_t_feat = relu_and_l2_norm_feat(self.feat_roi_align(t_feat.detach(), rois))
                own = torch.cat([torch.arange(n, device=s.device).to(s)[:, None], boxes], 1)
                roi_s_mask = self.mask_roi_align(s.detach()[:, None], own)[:, 0]
                roi_t_mask = self.mask_roi_align(t.detach()[:, None], own)[:, 0]
                iiu = torch.zeros((2 * n,) + tuple(s.shape[1:]), dtype=torch.float32, device=s.device)
            lvl_loss, lvl_num, _ = corr_level(self.solver, self.object_queues, self.first, roi_s_feat, roi_t_feat, roi_s_mask,
                                              roi_t_mask, boxes, klabels, valid, iiu, self.objbank_min_size, self.min_objs)
            total = total + lvl_loss
            num = num + lvl_num
            iiu = iiu.view(n, 2, *iiu.shape[1:])
            tf = target.float()
            enlarged = F.max_pool2d(tf[:, None], kernel_size=3, stride=1, padding=1)[:, 0]                  # :1128
            pseudo, _ = mean_field(((t + s) / 2)[:, None], tf[:, None], iiu, obj_img=img_inds)              # :1130-1132
            cropped = s * enlarged
            cropped = cropped * mean_field.gamma + cropped.detach() * (1 - mean_field.gamma)                # :1134
            x = cropped.flatten(1).float()                                                                  # dice_loss :542-550
            p = torch.where(valid[:, None], pseudo.flatten(1).float(), 0)
            ts = 1 - 2 * (x * p).sum(1) / ((x * x).sum(1) + 0.001 + (p * p).sum(1) + 0.001)
            out.append((torch.where(valid, ts, 0), valid))
        return total / (num + 1e-4), out

    def levels(self, s_ins_pred_list, t_ins_pred_list, img_ind_list, ins_labels, kernel_label_list, s_feat, t_feat, mean_field,
               use_ind_teacher=False):
        """Per level l: s_ins_pred_list[l] [n,H,W] student mask LOGITS (None: no object), t_ins_pred_list[l] the teacher's
        (ignored unless use_ind_teacher), img_ind_list[l] [n], ins_labels[l] [n,H,W] targets, kernel_label_list[l] [n];
        s_feat / t_feat [B,C,H,W]; mean_field: ONE ``MeanField`` over the batch's colour features (``obj_img`` selects the
        image; the reference keeps one module per image).  Returns (corr_loss / (num + 1e-4), [per-level dice terms [n_l] of
        the objects with a non-empty target]).  Compacting those lists costs one host synchronisation per level;
        ``levels_masked`` returns the same without it."""
        loss, per_level = self.levels_masked(s_ins_pred_list, t_ins_pred_list, img_ind_list, ins_labels, kernel_label_list,
                                             s_feat, t_feat, mean_field, use_ind_teacher)
        kept = [ts[valid] for ts, valid in per_level]
        return loss, [k for k in kept if k.numel()]
