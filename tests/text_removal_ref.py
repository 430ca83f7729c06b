"""torch restatement (CPU) of the text-removal stages of engine.TextRemovalStep that are not networks (DESIGN 5.2):

  * stage 3, text_mask:  sigmoid(logits) > 0.5, 3x3 max-pool (stride 1, padding 1), crop to the page: uint8 [n, 1, h, w];
  * stage 4, holes:      the mask as a {0, 255} image, > 0.4 * 255 (so: the set pixels), then the 10x10 dilation with the
                         anchor at (5, 5): output (y, x) is the max over rows y-5 .. y+4 and columns x-5 .. x+4, pixels outside
                         the page not taking part: bool [n, h, w];
  * stage 5, unet_input: valid = 1 - hole on the [hu, wu] grid (the padding is hole) and page * valid in fp32 (zero in the
                         padding): (uint8 [n, hu, wu], fp32 [n, 3, hu, wu]);
  * stage 7, composite:  valid ? page : fill, cropped to the page, fp32 [n, 3, h, w].

Shared by the CPU golden test and the GPU tests."""
import torch
import torch.nn.functional as F


def text_mask(logits: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """logits [n, 1, hs, ws] (any float dtype, any device) -> uint8 [n, 1, h, w] on the CPU."""
    x = logits.detach().float().cpu()[:, :1].contiguous()
    b = (torch.sigmoid(x) > 0.5).float()
    b = F.max_pool2d(b, 3, stride=1, padding=1)
    return b[:, :, :h, :w].to(torch.uint8).contiguous()


def holes(mask: torch.Tensor) -> torch.Tensor:
    """uint8 [n, 1, h, w] text mask (nonzero = text) -> bool [n, h, w] holes after the 10x10 dilation."""
    m = (mask.cpu()[:, 0] != 0).float()[:, None]
    # zero padding is neutral for a max over {0, 1}: the pixels outside the page never set a hole
    m = F.pad(m, (5, 4, 5, 4), value=0.0)
    return F.max_pool2d(m, 10, stride=1)[:, 0] > 0


def unet_input(mask: torch.Tensor, page: torch.Tensor, hu: int, wu: int):
    """(valid uint8 [n, hu, wu], corrupted fp32 [n, 3, hu, wu]) from the text mask and the fp32 page [n, 3, h, w]."""
    page = page.detach().float().cpu()
    n, _, h, w = page.shape
    hole = holes(mask)
    valid = torch.zeros((n, hu, wu), dtype=torch.uint8)
    valid[:, :h, :w] = (~hole).to(torch.uint8)
    corrupted = torch.zeros((n, 3, hu, wu), dtype=torch.float32)
    corrupted[:, :, :h, :w] = page * (~hole).float()[:, None]
    return valid, corrupted


def composite(fill: torch.Tensor, page: torch.Tensor, valid: torch.Tensor) -> torch.Tensor:
    """fp32 [n, 3, h, w]: the page where valid, the U-Net output `fill` [n, 3, hu, wu] elsewhere."""
    page = page.detach().float().cpu()
    n, _, h, w = page.shape
    keep = valid.cpu()[:, None, :h, :w] != 0
    return torch.where(keep, page, fill.detach().float().cpu()[:, :3, :h, :w])
