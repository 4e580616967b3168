"""TEST INFRASTRUCTURE ONLY -- numpy/scipy restatement of AnnotationLayerCOCO.forward (pylayers/pylayers/pylayers.py:
389-512), the COCO training input: decoded image -> zoomed, channel-swapped, mean-subtracted CHW blob; label map ->
one-hot cue planes and image tags; the epoch shuffle and the mirror draw from numpy.random in the reference's order.
Only tests/ and tools/ may import it.

Parity status: pinned against the reference's own class executed in place (oracle/ref_coco_layer.py ->
tests/golden/annot_coco_ref.npz, compared bit for bit in tests/test_annot_coco_cpu.py).
"""
import numpy as np
def coco_preprocess(image, label, new_size, mean, flip, ignore_label=255, K=81):
    """preprocess() of one image (pylayers.py:477-512) with the mirror draw given: flip = 1 or -1 (no mirror: 1).
    Returns (image (3,new_h,new_w) float64, cues (K,h,w) uint8, image_label (1,1,K) float64)."""
    from scipy.ndimage import zoom
    new_h, new_w = new_size
    image = np.array(image)                                                     # :483
    image = zoom(image.astype('float32'),                                       # :484-487
                 (new_h / float(image.shape[0]), new_w / float(image.shape[1]), 1.0), order=1)
    image = image[:, :, [2, 1, 0]]                                              # :489
    image = image - mean                                                        # :490
    image = image.transpose([2, 0, 1])                                          # :492
    h, w = label.shape                                                          # :494
    cues = np.zeros((K, h, w), dtype=np.uint8)                                  # :495
    for (x, y), v in np.ndenumerate(label):                                     # :496-498
        if not v == ignore_label:
            cues[v, x, y] = 1
    image = image[:, :, ::flip]                                                 # :502-503
    cues = cues[:, :, ::flip]
    unique_inst = np.unique(label)                                              # :505-507
    ignore_ind = np.where(unique_inst == ignore_label)[0]
    unique_inst = np.delete(unique_inst, ignore_ind)
    image_label = np.zeros((1, 1, K))                                           # :508-510
    for cat_id in unique_inst:
        image_label[0, 0, cat_id] = 1
    return image, cues, image_label


def annotation_coco_forward(read, indexlist, cur, root, batch_size, mean, new_size, is_mirror=False,
                            ignore_label=255, K=81):
    """AnnotationLayerCOCO.forward (pylayers.py:432-459) on `read(path, flag)` (cv2.imread's place; flag 1 = colour,
    0 = grey), drawing from numpy.random in the reference's order.  Shuffles `indexlist` in place like the reference.
    Returns (top0 (B,1,1,K), top1 (B,K,new_h//8+1,new_w//8+1), top2 (B,3,new_h,new_w) float32, the new _cur)."""
    new_h, new_w = new_size
    top0 = np.zeros((batch_size, 1, 1, K), np.float32)
    top1 = np.zeros((batch_size, K, new_h // 8 + 1, new_w // 8 + 1), np.float32)
    top2 = np.zeros((batch_size, 3, new_h, new_w), np.float32)
    for itt in range(batch_size):                                               # :433
        if cur == len(indexlist):                                               # :447-449
            cur = 0
            np.random.shuffle(indexlist)
        image_file_path, label_file_path = indexlist[cur]                       # :452-453
        image = read(root + image_file_path, 1)                                 # :456-457
        label = read(root + label_file_path, 0)
        cur += 1                                                                # :458
        flip = 1
        if is_mirror:                                                           # :500-501 (after the reads)
            flip = np.random.choice(2) * 2 - 1
        im, label_planes, image_label = coco_preprocess(image, label, new_size, mean, flip, ignore_label, K)
        top0[itt, ...] = image_label                                            # :438-440
        top1[itt, ...] = label_planes
        top2[itt, ...] = im
    return top0, top1, top2, cur
