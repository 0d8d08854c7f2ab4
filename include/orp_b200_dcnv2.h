/*
 * orp_b200_dcnv2.h - C ABI of liborp_b200.so, continued: the DCNv2 offset / mask split of ResNet backbones built with
 * dcn=dict(type='DCNv2') (mmdet/models/backbones/resnet.py:146-168).  Conventions (return codes, orp_last_error, device
 * pointers, asynchronous on `stream`) are those of orp_b200.h.
 */
#ifndef ORP_B200_DCNV2_H_
#define ORP_B200_DCNV2_H_

#ifdef __cplusplus
extern "C" {
#endif

/* ModulatedDeformConvPack.forward (mmdet/ops/dcn/deform_conv.py:411-419) after its conv_offset, deformable_groups = 1:
 *   om      device fp32 [pixels, 27], the conv_offset output in NHWC (channels o1 | o2 | mask logits, 9 each)
 *   offset  device fp32 [pixels, 18] = channels 0..17 in order (torch.cat((o1, o2), dim=1))
 *   mask    device fp32 [pixels, 9]  = sigmoid(channels 18..26), evaluated in fp64 and rounded once to fp32
 * These are the offset and mask layouts the deformable convolutions read (orp_tc_problem.offset / .mask,
 * orp_deform_conv2d_f32).  One launch; pixels == 0 is a no-op. */
int orp_dcnv2_offset_mask(const float *om, long long pixels, float *offset, float *mask, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_DCNV2_H_ */
