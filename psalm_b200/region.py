"""Host side of the region prompts (visual-prompt task, SURVEY.md section 8 f3).

`region_pooling` of the reference (visual_prompt_module/context_cluster.py:333-400) does two things: it DRAWS 256 sample
points per region mask on the host (`rand_sample_repeat`, context_cluster.py:31-40: torch.randint / torch.randperm on the
global CPU generator) and it samples + averages the projector's feature map at those points.  The second part is the
CUDA kernel `psalm_region_pool`; the first part is restated here with the same calls in the same order, so that a
caller who seeds the generator like the reference gets the reference's points."""
import torch

NUM_SAMPLE_POINT = 256   # llava_phi.py:162


def sample_region_points(region_masks, num_sample_point=NUM_SAMPLE_POINT):
    """region_masks [K,H,W] (bool / 0-1, host or device) -> [K, num_sample_point, 2] fp32 host tensor of normalised
    (y / H, x / W) positions of mask pixels: all of them plus random repeats when the mask is small, a random subset
    when it is large (context_cluster.py:31-40, :349-352)."""
    region_masks = region_masks.cpu()
    if region_masks.shape[0] == 0:
        return torch.zeros(0, num_sample_point, 2)
    wh = torch.tensor([region_masks[0].shape[0], region_masks[0].shape[1]])[None]
    out = []
    for m in region_masks:
        x = m.nonzero() / wh
        if x.shape[0] == 0:
            raise ValueError("empty region mask (the reference prints 'error' and then fails in torch.randint)")
        if x.shape[0] < num_sample_point:
            idx = torch.randint(0, x.shape[0], (num_sample_point - x.shape[0],))
            x = torch.cat((x, x[idx]), dim=0)
        elif x.shape[0] > num_sample_point:
            x = x[torch.randperm(x.shape[0])[:num_sample_point], :]
        out.append(x)
    return torch.stack(out).float()


def draw_point_indices(counts, num_sample_point=NUM_SAMPLE_POINT):
    """The random part of `sample_region_points` for masks with `counts` set pixels: [K, num_sample_point] int32 indices
    into each mask's `nonzero()` rows, drawn with the same calls in the same order on the global CPU generator, so that
    `m.nonzero()[idx] / wh` equals `sample_region_points` from the same generator state.  The masks themselves stay on the
    device (kernels.region_points_gather turns the indices into points)."""
    out = []
    for n in counts:
        n = int(n)
        if n == 0:
            raise ValueError("empty region mask (the reference prints 'error' and then fails in torch.randint)")
        if n < num_sample_point:
            idx = torch.cat((torch.arange(n), torch.randint(0, n, (num_sample_point - n,))))
        elif n > num_sample_point:
            idx = torch.randperm(n)[:num_sample_point]
        else:
            idx = torch.arange(n)
        out.append(idx)
    return torch.stack(out).to(torch.int32)


def region_inputs(seg_info, region_points=None, attr="region_masks"):
    """seg_info: list of dicts with 'instances' (`.region_masks.tensor` [K,H,W], llava_phi.py:792; the DAVIS variant reads
    `.vp_region_masks`, :1664) -> (points [R,P,2] fp32, region_image [R] int32, counts).  `region_points`: optional
    per-sample list of pre-drawn points."""
    pts, img, counts = [], [], []
    for b, info in enumerate(seg_info):
        p = region_points[b] if region_points is not None else sample_region_points(getattr(info["instances"], attr).tensor)
        pts.append(p.float().cpu())
        img += [b] * p.shape[0]
        counts.append(int(p.shape[0]))
    return torch.cat(pts, 0).contiguous(), torch.tensor(img, dtype=torch.int32), tuple(counts)
