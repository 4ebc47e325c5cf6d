"""Backbone factory with the reference's signature (backbone/select_backbone.py:4-16)."""
from .s3dg import S3D
from .resnet_2d3d import r2d3d50


def select_backbone(network, first_channel=3):
    """-> (module, {'feature_size': int}). 's3d', 's3dg' (S3D with feature gating) and 'r50' run on the sm_90a engine;
    unknown names raise NotImplementedError as in the reference."""
    param = {'feature_size': 1024}
    if network == 's3d':
        model = S3D(input_channel=first_channel)
    elif network == 's3dg':
        model = S3D(input_channel=first_channel, gating=True)
    elif network == 'r50':
        param['feature_size'] = 2048
        model = r2d3d50(input_channel=first_channel)
    else:
        raise NotImplementedError("backbone %r is not available in coclr_b200 (supported: 's3d', 's3dg', 'r50')" % (network,))
    return model, param
