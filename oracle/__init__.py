"""oracle/ -- TEST INFRASTRUCTURE ONLY.

CPU restatement of the partial-convolution hot path of
yu45020/Text_Segmentation_Image_Inpainting.  Nothing in the product package
(`text_segmentation_image_inpainting_b200/`) imports from here.  The only
legal importers are `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py`, and there only as the
checker / the timed CPU baseline -- never as the thing shipped.

Parity status: PINNED.  The reference is pure Python over ATen; it imports and
runs in the build container (torch 2.11 CPU).  `tests/golden/make_golden.py`
runs the reference's own modules there and commits the outputs as fixtures;
`tests/test_oracle_golden.py` checks this restatement against those fixtures
bit-for-bit (same ATen ops, same order).

Where the arithmetic lives: torch.nn.functional.conv2d / batch_norm /
interpolate (ATen, third-party, un-vendored; the reference pins no version --
the installed torch 2.11.0 CPU build is the oracle's arithmetic).  The plain-C
file `pconv_box.c` restates the same algorithm with direct loops (box-sum
form of the all-ones mask convolution) as an ATen-independent cross-check.
"""
