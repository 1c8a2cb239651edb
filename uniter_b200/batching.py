"""Host-side batching for the hot path (SURVEY.md §8f-3): the reference's token-bucket sampler and
collate functions restated without their LMDB / horovod / toolz dependencies, emitting the SAME
padded batch dict the reference models consume plus the host-known bookkeeping that lets the
GPU path run without a single device->host read:

* ``TokenBucketSampler``  — data/sampler.py:17-60, same algorithm and the same use of the global
  ``random`` state (so ``random.seed(s)`` reproduces the reference's batches exactly); an explicit
  ``random.Random`` can be injected instead.
* ``vqa_collate`` / ``mlm_collate`` — data/vqa.py:44-71, data/mlm.py:96-136 (``pad_tensors`` and
  ``get_gather_index`` from data/data.py:255-279).  Extra keys (ignored by the reference heads):
  ``txt_lens``, ``num_bbs`` (python lists), ``cu_seqlens`` (int32 [B+1], packed-row offsets of each
  sample), and for MLM ``mlm_index`` / ``mlm_targets`` (flat b*L+j positions and labels of the
  masked tokens, in the order of the reference's boolean-mask selection, model/pretrain.py:129-133).
* ``re_collate`` / ``re_eval_collate`` — data/re.py:146-188, :251-295, plus ``re_index`` / ``re_seg``, the
  flat positions of the region rows and each sample's start and count in them (``re_region_index``).
* ``itm_ot_collate`` — data/itm.py:128-183: ITM pairs with the word-region alignment inputs (``ot_inputs``,
  uint8 pads), plus ``ot_txt_lens`` (int32 text lengths) and ``ot_pos_index`` / ``ot_neg_index`` (int64
  positions of the positive / negative pairs), with which the ITM step reads nothing from the device.
* ``vcr_collate`` / ``vcr_eval_collate`` — data/vcr.py:162-196, :262-300: every question contributes one
  sequence per choice (4 answers; for eval also the 16 rationale sequences), flattened in order.
* ``DevicePrefetcher`` — data/loader.py:86-141 (side-stream H2D of pinned batches, joined with
  ``wait_stream`` + ``record_stream``), additionally registering the per-sample lengths of the
  device attention mask with the model (``register_lengths``) so forward() never syncs.
"""
import random as _random

import torch
from torch.nn.utils.rnn import pad_sequence

from .synth import get_gather_index


class TokenBucketSampler(object):
    """Batches of sample ids whose PADDED size (max_len x batch) stays below `batch_size` tokens;
    batch length is a multiple of `size_multiple` except possibly the last one of a bucket."""

    def __init__(self, lens, bucket_size, batch_size, droplast=False, size_multiple=8, rng=None):
        self._lens = lens
        self._max_tok = batch_size
        self._bucket_size = bucket_size
        self._droplast = droplast
        self._size_mul = size_multiple
        self._rng = rng if rng is not None else _random

    def _create_ids(self):
        return list(range(len(self._lens)))

    def _sort_fn(self, i):
        return self._lens[i]

    def __iter__(self):
        ids = self._create_ids()
        self._rng.shuffle(ids)
        buckets = [sorted(ids[i:i + self._bucket_size], key=self._sort_fn, reverse=True)
                   for i in range(0, len(ids), self._bucket_size)]
        batches = []
        for bucket in buckets:
            max_len = 0
            batch_indices = []
            for k in range(0, len(bucket), self._size_mul):       # cytoolz.partition_all
                indices = bucket[k:k + self._size_mul]
                max_len = max(max_len, max(self._lens[i] for i in indices))
                if max_len * (len(batch_indices) + self._size_mul) > self._max_tok:
                    if not batch_indices:
                        raise ValueError("max_tokens too small / max_seq_len too long")
                    assert len(batch_indices) % self._size_mul == 0
                    batches.append(batch_indices)
                    batch_indices = list(indices)
                else:
                    batch_indices.extend(indices)
            if not self._droplast and batch_indices:
                batches.append(batch_indices)
        self._rng.shuffle(batches)
        return iter(batches)

    def __len__(self):
        raise ValueError("NOT supported. This has some randomness across epochs")


def pad_tensors(tensors, lens=None, pad=0):
    """B x [T, ...] -> [B, max T, ...] (data/data.py:255-268)."""
    if lens is None:
        lens = [t.size(0) for t in tensors]
    max_len = max(lens)
    bs = len(tensors)
    hid = tensors[0].size(-1)
    output = torch.zeros(bs, max_len, hid, dtype=tensors[0].dtype)
    if pad:
        output.fill_(pad)
    for i, (t, l) in enumerate(zip(tensors, lens)):
        output[i, :l, ...] = t
    return output


def _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks):
    txt_lens = [i.size(0) for i in input_ids]
    input_ids = pad_sequence(input_ids, batch_first=True, padding_value=0)
    position_ids = torch.arange(0, input_ids.size(1), dtype=torch.long).unsqueeze(0)
    attn_masks = pad_sequence(attn_masks, batch_first=True, padding_value=0)
    num_bbs = [f.size(0) for f in img_feats]
    img_feat = pad_tensors(img_feats, num_bbs)
    img_pos_feat = pad_tensors(img_pos_feats, num_bbs)
    bs, max_tl = input_ids.size()
    out_size = attn_masks.size(1)
    gather_index = get_gather_index(txt_lens, num_bbs, bs, max_tl, out_size)
    cu = [0]
    for tl, nbb in zip(txt_lens, num_bbs):
        cu.append(cu[-1] + tl + nbb)
    return {"input_ids": input_ids, "position_ids": position_ids, "img_feat": img_feat,
            "img_pos_feat": img_pos_feat, "attn_masks": attn_masks, "gather_index": gather_index,
            "txt_lens": txt_lens, "num_bbs": num_bbs,
            "cu_seqlens": torch.tensor(cu, dtype=torch.int32)}


def vqa_collate(inputs):
    """inputs: list of (input_ids [tl], img_feat [nbb, D], img_pos_feat [nbb, 7], attn_masks
    [tl + nbb], target [answers]) — data/vqa.py:44-71."""
    input_ids, img_feats, img_pos_feats, attn_masks, targets = map(list, zip(*inputs))
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    batch["targets"] = torch.stack(targets, dim=0)
    return batch


def mlm_collate(inputs):
    """inputs: list of (input_ids, img_feat, img_pos_feat, attn_masks, txt_labels [tl], -1 = not
    masked) — data/mlm.py:96-136."""
    input_ids, img_feats, img_pos_feats, attn_masks, txt_labels = map(list, zip(*inputs))
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    txt_labels = pad_sequence(txt_labels, batch_first=True, padding_value=-1)
    batch["txt_labels"] = txt_labels
    L = batch["attn_masks"].size(1)
    pos = (txt_labels != -1).nonzero(as_tuple=False)
    batch["mlm_index"] = (pos[:, 0] * L + pos[:, 1]).contiguous()
    batch["mlm_targets"] = txt_labels[pos[:, 0], pos[:, 1]].contiguous()
    return batch


def re_region_index(txt_lens, num_bbs, L, multiple=64):
    """Where the image regions of a referring-expression batch sit (model/re.py:129-157,
    `_get_image_hidden`): flat positions b * L + txt_lens[b] + k of the padded [B, L] layout, padded
    with the "no row" position B * L to a multiple of `multiple` (int64), and int32 [2, B] with the
    start of each sample's regions in that list and their count."""
    B = len(txt_lens)
    flat, starts = [], []
    for b, (tl, nbb) in enumerate(zip(txt_lens, num_bbs)):
        starts.append(len(flat))
        flat.extend(range(b * L + tl, b * L + tl + nbb))
    n = max((len(flat) + multiple - 1) // multiple * multiple, multiple)
    flat.extend([B * L] * (n - len(flat)))
    return torch.tensor(flat, dtype=torch.long), torch.tensor([starts, list(num_bbs)], dtype=torch.int32)


def _re_fields(input_ids, img_feats, img_pos_feats, attn_masks, obj_masks):
    """data/re.py:146-188 without the targets: the joint fields, obj_masks padded with 1 (uint8, as the
    datasets build it), and the region index of re_region_index as `re_index` / `re_seg`."""
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    if min(batch["num_bbs"]) < 1:
        raise ValueError("every sample needs at least one region, got num_bbs %s" % batch["num_bbs"])
    batch["obj_masks"] = pad_sequence(obj_masks, batch_first=True, padding_value=1)
    batch["re_index"], batch["re_seg"] = re_region_index(batch["txt_lens"], batch["num_bbs"],
                                                         batch["attn_masks"].size(1))
    return batch


def re_collate(inputs):
    """inputs: list of (input_ids, img_feat, img_pos_feat, attn_masks, obj_masks [nbb] uint8, target [1])
    — data/re.py:146-188 (ReDataset)."""
    input_ids, img_feats, img_pos_feats, attn_masks, obj_masks, targets = map(list, zip(*inputs))
    batch = _re_fields(input_ids, img_feats, img_pos_feats, attn_masks, obj_masks)
    targets = torch.stack(targets, dim=0)
    for t, nbb in zip(targets.view(-1).tolist(), batch["num_bbs"]):
        if not 0 <= t < nbb:
            raise ValueError("target %d outside [0, %d)" % (t, nbb))
    batch["targets"] = targets
    return batch


def re_eval_collate(inputs):
    """inputs: list of (input_ids, img_feat, img_pos_feat, attn_masks, obj_masks, tgt_box, obj_boxes,
    sent_id) — data/re.py:251-295 (ReEvalDataset)."""
    (input_ids, img_feats, img_pos_feats, attn_masks, obj_masks, tgt_box, obj_boxes,
     sent_ids) = map(list, zip(*inputs))
    batch = _re_fields(input_ids, img_feats, img_pos_feats, attn_masks, obj_masks)
    batch["tgt_box"], batch["obj_boxes"], batch["sent_ids"] = tgt_box, obj_boxes, sent_ids
    return batch


def _ot_pad(lens, max_len):
    pad = torch.zeros(len(lens), max_len, dtype=torch.uint8)
    for i, n in enumerate(lens):
        pad[i, n:] = 1
    return pad


def itm_ot_collate(inputs):
    """inputs: list of (input_ids, img_feat, img_pos_feat, attn_masks, target [1]) — data/itm.py:145-183
    (ItmDataset with itm_ot_lambda > 0).  ot_scatter maps position j < txt_len of pair i to text slot j
    and j >= txt_len to image slot j - txt_len (data/itm.py:128-135)."""
    input_ids, img_feats, img_pos_feats, attn_masks, targets = map(list, zip(*inputs))
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    targets = torch.cat(targets, dim=0)
    txt_lens, num_bbs = batch["txt_lens"], batch["num_bbs"]
    joint_len, max_tl = batch["attn_masks"].size(1), max(txt_lens)
    ot_scatter = torch.arange(0, joint_len, dtype=torch.long).unsqueeze(0).repeat(len(txt_lens), 1)
    for i, tl in enumerate(txt_lens):
        ot_scatter[i, tl:] = torch.arange(max_tl, max_tl + joint_len - tl, dtype=torch.long)
    batch["targets"] = targets
    batch["ot_inputs"] = {"ot_scatter": ot_scatter, "scatter_max": ot_scatter.max().item(),
                          "txt_pad": _ot_pad(txt_lens, max_tl), "img_pad": _ot_pad(num_bbs, max(num_bbs))}
    batch["ot_txt_lens"] = torch.tensor(txt_lens, dtype=torch.int32)
    t = targets.tolist()
    batch["ot_pos_index"] = torch.tensor([i for i, v in enumerate(t) if v == 1], dtype=torch.long)
    batch["ot_neg_index"] = torch.tensor([i for i, v in enumerate(t) if v == 0], dtype=torch.long)
    return batch


def _vcr_fields(input_ids, txt_type_ids, img_feats, img_pos_feats, attn_masks):
    """The joint fields plus txt_type_ids padded with 0 (data/vcr.py:166-168)."""
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    out = {"input_ids": batch.pop("input_ids"),
           "txt_type_ids": pad_sequence(txt_type_ids, batch_first=True, padding_value=0)}
    out.update(batch)
    return out


def vcr_collate(inputs):
    """inputs: one tuple per question of (input_ids, txt_type_ids, img_feat, img_pos_feat, attn_masks,
    target [1]) per choice — data/vcr.py:162-196 (VcrDataset).  targets: [n_choices_total, 1]."""
    (input_ids, txt_type_ids, img_feats, img_pos_feats, attn_masks,
     targets) = map(list, zip(*[c for q in inputs for c in q]))
    batch = _vcr_fields(input_ids, txt_type_ids, img_feats, img_pos_feats, attn_masks)
    batch["targets"] = torch.stack(targets, dim=0)
    return batch


def vcr_eval_collate(inputs):
    """inputs: one (choices, qid, qa_target [1], qar_target [1]) per question, choices a tuple of
    (input_ids, txt_type_ids, img_feat, img_pos_feat, attn_masks) — data/vcr.py:262-300 (VcrEvalDataset)."""
    (input_ids, txt_type_ids, img_feats, img_pos_feats,
     attn_masks) = map(list, zip(*[c for outs, _, _, _ in inputs for c in outs]))
    batch = _vcr_fields(input_ids, txt_type_ids, img_feats, img_pos_feats, attn_masks)
    batch["qa_targets"] = torch.stack([t for _, _, t, _ in inputs], dim=0)
    batch["qar_targets"] = torch.stack([t for _, _, _, t in inputs], dim=0)
    batch["qids"] = [qid for _, qid, _, _ in inputs]
    return batch


class DevicePrefetcher(object):
    """Iterate a loader of collated batches with the next batch's H2D copy overlapped on a side
    stream (data/loader.py:86-141).  Tensors are pinned here if the loader did not pin them."""

    def __init__(self, loader, device=None):
        self.loader = loader
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        self.stream = torch.cuda.Stream(self.device)

    def __len__(self):
        return len(self.loader)

    def _to_device(self, batch):
        from .model import register_lengths
        out = {}
        with torch.cuda.stream(self.stream):
            for k, v in batch.items():
                if torch.is_tensor(v):
                    if not v.is_pinned():
                        v = v.pin_memory()
                    out[k] = v.to(self.device, non_blocking=True)
                else:
                    out[k] = v
        if "txt_lens" in batch and "num_bbs" in batch and "attn_masks" in out:
            register_lengths(out["attn_masks"], [a + b for a, b in zip(batch["txt_lens"], batch["num_bbs"])],
                             prefix=True)
        return out

    def __iter__(self):
        it = iter(self.loader)
        nxt = None
        try:
            nxt = self._to_device(next(it))
        except StopIteration:
            return
        while nxt is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.stream)
            batch = nxt
            for v in batch.values():
                if torch.is_tensor(v):
                    v.record_stream(torch.cuda.current_stream(self.device))
            try:
                nxt = self._to_device(next(it))
            except StopIteration:
                nxt = None
            yield batch


# ============================================================================ MRM collates
def _mrm_fields(input_ids, img_feats, img_pos_feats, attn_masks, img_masks, img_mask_tgts):
    """Common part of data/mrm.py:76-123 (mrfr_collate) and :176-227 (mrc_collate): pad, build the
    joint fields, extract the masked regions' targets, zero the masked input features."""
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    img_masks = pad_sequence(img_masks, batch_first=True, padding_value=0)
    img_mask_tgt = pad_sequence(img_mask_tgts, batch_first=True, padding_value=0)
    batch["img_masks"] = img_masks
    batch["img_mask_tgt"] = img_mask_tgt
    # host-side compaction of the masked positions (flat b * L + j), the fixed-shape stand-in for
    # `_compute_masked_hidden` (model/pretrain.py:129-133)
    L = batch["attn_masks"].size(1)
    pos = img_mask_tgt.nonzero(as_tuple=False)
    batch["mrm_index"] = (pos[:, 0] * L + pos[:, 1]).contiguous()
    return batch, img_masks


def mrfr_collate(inputs):
    """inputs: list of (input_ids, img_feat, img_pos_feat, attn_masks, img_mask [nbb] bool,
    img_mask_tgt [tl + nbb]) — data/mrm.py:76-123."""
    input_ids, img_feats, img_pos_feats, attn_masks, img_masks, img_mask_tgts = map(list, zip(*inputs))
    batch, img_masks = _mrm_fields(input_ids, img_feats, img_pos_feats, attn_masks, img_masks, img_mask_tgts)
    img_feat = batch["img_feat"]
    ext = img_masks.unsqueeze(-1).expand_as(img_feat)
    batch["feat_targets"] = img_feat[ext].contiguous().view(-1, img_feat.size(-1))   # data/mrm.py:29-34
    batch["img_feat"] = img_feat.data.masked_fill(ext, 0)                            # :37-40
    return batch


def mrc_collate(inputs):
    """inputs: list of (input_ids, img_feat, img_pos_feat, img_soft_labels [nbb, C], attn_masks,
    img_mask, img_mask_tgt) — data/mrm.py:176-227."""
    (input_ids, img_feats, img_pos_feats, img_soft_labels, attn_masks, img_masks,
     img_mask_tgts) = map(list, zip(*inputs))
    batch, img_masks = _mrm_fields(input_ids, img_feats, img_pos_feats, attn_masks, img_masks, img_mask_tgts)
    num_bbs = batch["num_bbs"]
    img_soft_label = pad_tensors(img_soft_labels, num_bbs)
    ext_l = img_masks.unsqueeze(-1).expand_as(img_soft_label)
    batch["label_targets"] = img_soft_label[ext_l].contiguous().view(-1, img_soft_label.size(-1))
    ext = img_masks.unsqueeze(-1).expand_as(batch["img_feat"])
    batch["img_feat"] = batch["img_feat"].data.masked_fill(ext, 0)
    return batch


# ============================================================================ ITM ranking batches
def sample_negative(sample_pool, ground_truths, num_sample, rng=None):
    """data/itm.py:36-46 — random.sample and retry until disjoint from the ground truths."""
    rng = rng if rng is not None else _random
    outputs = ground_truths[:1]
    while set(outputs) & set(ground_truths):
        outputs = rng.sample(sample_pool, num_sample)
    return outputs


def itm_rank_collate(inputs):
    """inputs: list (one entry per anchor) of lists of (input_ids, img_feat, img_pos_feat,
    attn_masks) — positive pair first, then the negatives (data/itm.py:240-269)."""
    flat = [t for sample in inputs for t in sample]
    input_ids, img_feats, img_pos_feats, attn_masks = map(list, zip(*flat))
    batch = _joint_fields(input_ids, img_feats, img_pos_feats, attn_masks)
    sample_size = len(inputs[0])
    assert all(sample_size == len(i) for i in inputs)
    batch["sample_size"] = sample_size
    return batch


def hard_neg_batch_from_text(input_ids, img_feats, img_pos_feats):
    """One text against 1 + N images, ground truth first (ItmRankDatasetHardNegFromText.__getitem__,
    data/itm.py:282-320).  input_ids [tl]; img_feats / img_pos_feats: lists of [nbb_i, D] / [nbb_i, 7]."""
    input_ids = input_ids.unsqueeze(0)
    position_ids = torch.arange(0, input_ids.size(1), dtype=torch.long).unsqueeze(0)
    num_bbs = [f.size(0) for f in img_feats]
    img_feat = pad_tensors(img_feats, num_bbs)
    img_pos_feat = pad_tensors(img_pos_feats, num_bbs)
    tl = input_ids.size(1)
    n = len(img_feats)
    attn_masks = torch.zeros(n, max(num_bbs) + tl).long()
    for i, nbb in enumerate(num_bbs):
        attn_masks.data[i, :tl + nbb].fill_(1)
    gather_index = get_gather_index([tl] * n, num_bbs, n, tl, attn_masks.size(1))
    return {"input_ids": input_ids, "position_ids": position_ids, "img_feat": img_feat,
            "img_pos_feat": img_pos_feat, "attn_masks": attn_masks, "gather_index": gather_index,
            "txt_lens": [tl] * n, "num_bbs": num_bbs}


def hard_neg_batch_from_image(img_feat, img_pos_feat, all_input_ids):
    """One image against 1 + N texts, ground truth first (ItmRankDatasetHardNegFromImage.__getitem__,
    data/itm.py:323-369).  Reproduces the reference's gather_index EXACTLY, including its use of the
    loop variable `tl` left over from the last text as `max_len` (data/itm.py:356-361): image slots
    then index rows relative to the LAST text's length instead of the padded text length — the
    drop-in encoder honours whatever index arrives (SURVEY.md §8a E3)."""
    nbb = img_feat.size(0)
    img_feat = img_feat.unsqueeze(0)
    img_pos_feat = img_pos_feat.unsqueeze(0)
    txt_lens = [len(i) for i in all_input_ids]
    input_ids = pad_sequence(all_input_ids, batch_first=True, padding_value=0)
    position_ids = torch.arange(0, input_ids.size(1), dtype=torch.long).unsqueeze(0)
    n = len(all_input_ids)
    attn_masks = torch.zeros(n, max(txt_lens) + nbb).long()
    for i, tl in enumerate(txt_lens):
        attn_masks.data[i, :tl + nbb].fill_(1)
    stale_tl = txt_lens[-1]
    gather_index = get_gather_index(txt_lens, [nbb] * n, n, stale_tl, attn_masks.size(1))
    return {"input_ids": input_ids, "position_ids": position_ids, "img_feat": img_feat,
            "img_pos_feat": img_pos_feat, "attn_masks": attn_masks, "gather_index": gather_index,
            "txt_lens": txt_lens, "num_bbs": [nbb] * n}


def itm_rank_hn_collate(inputs):
    """data/itm.py:372-374."""
    assert len(inputs) == 1
    return inputs[0]


def _img_feat_of(img_db, fname):
    """DetectFeatTxtTokDataset._get_img_feat (data/data.py:247-251): 7-d box = (x1,y1,x2,y2,w,h,w*h)."""
    img_feat, bb = img_db[fname]
    img_bb = torch.cat([bb, bb[:, 4:5] * bb[:, 5:]], dim=-1)
    return img_feat, img_bb, img_feat.size(0)


class ItmRankDatasetHardNegFromText(object):
    """data/itm.py:282-320 over duck-typed stores: `txt_db[id]['input_ids']` (list of token ids),
    `txt_db.combine_inputs(ids)` ([CLS] ids [SEP] tensor), `img_db[fname] -> (feat [n, D], bb [n, 6])`.
    Negatives are drawn with the global `random` state exactly like the reference."""

    def __init__(self, txt_db, img_db, ids, txt2img, img2txts, neg_sample_size=1, rng=None):
        assert neg_sample_size > 0, "need at least 1 negative sample"
        self.txt_db, self.img_db, self.ids = txt_db, img_db, list(ids)
        self.txt2img = {id_: txt2img[id_] for id_ in self.ids}
        self.img2txts = img2txts
        self.img_name_list = list(self.img2txts.keys())
        self.neg_sample_size = neg_sample_size
        self.rng = rng

    def __len__(self):
        return len(self.ids)

    def __getitem__(self, i):
        gt_txt_id = self.ids[i]
        gt_img_fname = self.txt2img[gt_txt_id]
        input_ids = self.txt_db.combine_inputs(self.txt_db[gt_txt_id]["input_ids"])
        neg_img_ids = sample_negative(self.img_name_list, [gt_img_fname], self.neg_sample_size, self.rng)
        feats, boxes = [], []
        for fname in [gt_img_fname] + neg_img_ids:
            f, b, _ = _img_feat_of(self.img_db, fname)
            feats.append(f)
            boxes.append(b)
        return hard_neg_batch_from_text(input_ids, feats, boxes)


class ItmRankDatasetHardNegFromImage(object):
    """data/itm.py:323-369 (see hard_neg_batch_from_image for the gather_index quirk it keeps)."""

    def __init__(self, txt_db, img_db, ids, txt2img, img2txts, neg_sample_size=1, rng=None):
        assert neg_sample_size > 0, "need at least 1 negative sample"
        self.txt_db, self.img_db, self.ids = txt_db, img_db, list(ids)
        self.txt2img = {id_: txt2img[id_] for id_ in self.ids}
        self.img2txts = img2txts
        self.txt_name_list = list(self.txt2img.keys())
        self.neg_sample_size = neg_sample_size
        self.rng = rng

    def __len__(self):
        return len(self.ids)

    def __getitem__(self, i):
        gt_txt_id = self.ids[i]
        gt_img_id = self.txt2img[gt_txt_id]
        gt_txt_ids = self.img2txts[gt_img_id]
        img_feat, img_pos_feat, _ = _img_feat_of(self.img_db, gt_img_id)
        neg_txt_ids = sample_negative(self.txt_name_list, gt_txt_ids, self.neg_sample_size, self.rng)
        all_inputs = [self.txt_db.combine_inputs(self.txt_db[t]["input_ids"]) for t in [gt_txt_id] + neg_txt_ids]
        return hard_neg_batch_from_image(img_feat, img_pos_feat, all_inputs)
