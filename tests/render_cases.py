"""The golden render cases: one table shared by tests/golden/make_golden.py (which renders them with the
unmodified reference), tests/test_oracle_golden.py (oracle vs those images) and tests/test_gpu_parity.py /
tests/test_dropin_plugin.py (CUDA path and drop-in binary vs those images)."""

# name: (n_tris, materials, xres, yres, spp, maxdepth, light sample strategy, n_lights)
RENDERS = {
    "matte": (3000, ("matte",), 40, 32, 8, 5, "uniform", None),
    "four": (3000, ("matte", "glass", "metal", "plastic"), 40, 32, 8, 5, "uniform", None),
    "power16": (3000, ("matte", "glass", "metal", "plastic"), 32, 32, 4, 16, "power", 16),
    # thin-lens camera, two-sided lights, ReverseOrientation on the glass and plastic meshes
    "lens_flip": (3000, ("matte", "glass", "metal", "plastic"), 36, 24, 8, 6, "uniform", None),
    # pbrt's default light sample strategy (SpatialLightDistribution), 10 and 16 lights
    "spatial": (3000, ("matte", "glass", "metal", "plastic"), 40, 32, 8, 5, "spatial", None),
    "spatial16": (3000, ("matte", "plastic"), 32, 32, 4, 8, "spatial", 16),
    # per-vertex shading normals (matte + metal meshes) and uvs (matte + plastic meshes), flipped plastic
    "normals_uv": (3000, ("matte", "glass", "metal", "plastic"), 40, 32, 8, 6, "spatial", None),
    # film crop window (sampler built from the cropped sample bounds), film scale, maxsampleluminance
    "crop": (3000, ("matte", "glass", "metal", "plastic"), 70, 50, 4, 5, "uniform", None),
    # non-default lobes of the four materials: OrenNayar matte (sigma 30), rough glass (microfacet reflection +
    # transmission)
    "rough": (3000, ("matte_rough", "glass_rough", "metal", "plastic"), 40, 32, 8, 8, "spatial", None),
    # HaltonSampler (pbrt's default sampler): non-power-of-two sample counts, cropped sample bounds
    "halton": (3000, ("matte", "glass", "metal", "plastic"), 40, 32, 6, 5, "spatial", None),
    "halton_crop": (3000, ("matte", "plastic"), 70, 50, 3, 5, "uniform", None),
    # Sphere shapes: two sphere area lights (one under a uniform scale) next to the 10 quad lights, a glass
    # sphere, a plastic ellipsoid under a handedness-swapping scale, a matte sphere with ReverseOrientation
    "spheres": (3000, ("matte", "glass", "metal", "plastic"), 48, 40, 8, 6, "spatial", None),
    # the only light is a sphere (the situation of scenes/killeroo-simple.pbrt), Halton sampler
    "sphere_light": (3000, ("matte", "plastic"), 40, 32, 6, 5, "spatial", 0),
    "sphere_power": (3000, ("matte", "glass_rough"), 40, 32, 4, 7, "power", 4),
    # partial spheres (zmin / zmax / phimax clipping: std::atan2, second root), one of them an area light
    "sphere_partial": (3000, ("matte", "plastic"), 48, 40, 8, 5, "spatial", 4),
    # object instancing (TransformedPrimitive): two objects, five instances (one at the identity, one mirrored)
    "instances": (2000, ("matte", "glass", "metal", "plastic"), 48, 40, 8, 6, "spatial", None),
    # instances under rotations about oblique axes: T S R (non-orthogonal linear part), T R S, R T S, mirrored and rotated,
    # one at the identity -- full instance matrices for the normal transform, the error offset and the world boxes
    "instances_affine": (2000, ("matte", "glass", "metal", "plastic"), 48, 40, 8, 6, "spatial", None),
    # MirrorMaterial (SpecularReflection + FresnelNoOp) next to glass: long specular chains
    "mirror": (3000, ("matte", "mirror", "glass", "plastic"), 40, 32, 8, 8, "spatial", None),
    # delta lights (point, spot, distant) next to the area lights: no MIS branch, Light::Power / Sample_Li per kind
    "delta_lights": (3000, ("matte", "glass", "metal", "plastic"), 40, 32, 8, 5, "spatial", 4),
    "delta_power": (3000, ("matte", "plastic"), 40, 32, 4, 5, "power", 0),
    # the reference's own known-answer scenes (src/tests/analytic_scenes.cpp:69-160): camera inside a unit sphere with
    # Kd 0.5 (reverse orientation) lit by a point light of intensity pi at the centre, by four of pi/4, or emitting 0.5
    # itself -- the radiance is 1 everywhere; PathIntegrator depth 8, 10x10 pixels, 256 samples, fov 45
    "analytic_point": (0, ("matte",), 10, 10, 256, 8, "spatial", 0),
    "analytic_4points": (0, ("matte",), 10, 10, 256, 8, "spatial", 0),
    "analytic_area": (0, ("matte",), 10, 10, 256, 8, "spatial", 0),
    # pixel filters wider than the box (Film::filterTable weights, samples outside the film, tile aprons of 2-4
    # pixels); the reference image is rendered with --nthreads 1 so that its tile merge order is defined
    "filter_gaussian": (3000, ("matte", "glass", "metal", "plastic"), 40, 36, 4, 5, "spatial", None),
    "filter_mitchell": (3000, ("matte", "plastic"), 37, 33, 4, 5, "uniform", None),
    "filter_sinc": (3000, ("matte", "plastic"), 40, 32, 3, 5, "uniform", None),
    "filter_aniso_crop": (3000, ("matte", "metal"), 70, 50, 4, 5, "uniform", None),
    "filter_triangle": (3000, ("matte", "glass"), 33, 35, 4, 5, "power", None),
    "filter_box1": (3000, ("matte", "plastic"), 40, 32, 4, 5, "uniform", None),
}
EXTRA = {"lens_flip": dict(scene=dict(two_sided=True, reverse_orientation=(1, 3)),
                           camera=dict(lens_radius=0.05, focal_distance=4.5)),
         "normals_uv": dict(scene=dict(shading_normals=(0, 2), uvs=(0, 3), reverse_orientation=(3,))),
         "crop": dict(camera=dict(crop_window=(0.21, 0.83, 0.1, 0.74), film_scale=2.0, max_sample_luminance=9.0)),
         "halton": dict(camera=dict(sampler="halton")),
         "halton_crop": dict(camera=dict(sampler="halton", crop_window=(0.21, 0.83, 0.1, 0.74))),
         "spheres": dict(scene=dict(spheres=(
             dict(center=(1.2, 1.8, -1.5), radius=0.35, emit=60.0),
             dict(center=(-2.0, 0.5, -2.5), radius=0.2, emit=90.0, scale=(1.5, 1.5, 1.5)),
             dict(center=(0.1, 0.0, -2.2), radius=0.45, material="glass"),
             dict(center=(-0.9, -0.6, -2.0), radius=0.4, material="plastic", scale=(1.3, 0.7, -1.1)),
             dict(center=(0.9, -0.7, -1.9), radius=0.3, material="matte", reverse_orientation=True)))),
         "sphere_partial": dict(scene=dict(spheres=(
             dict(center=(0.1, 0.1, -2.2), radius=0.6, material="plastic", zmin=-0.3, zmax=0.45, phimax=250.0),
             dict(center=(-1.0, -0.6, -2.0), radius=0.5, material="matte", scale=(1.2, 0.8, 1.0), phimax=200.0,
                  reverse_orientation=True),
             dict(center=(1.1, 0.6, -1.8), radius=0.4, emit=80.0, zmin=-0.1, two_sided=True)))),
         "instances": dict(scene=dict(
             objects=(dict(n_tris=400, seed=5, material="plastic", size=0.35), dict(n_tris=150, seed=9, material="glass", size=0.5)),
             instances=(dict(object=0, center=(0.0, 0.0, -2.4)), dict(object=0, center=(1.2, 0.8, -2.0), scale=(0.7, 1.4, 1.0)),
                        dict(object=1, center=(-1.1, -0.7, -2.2), scale=(1.0, 1.0, -1.3)), dict(object=1),
                        dict(object=0, center=(-1.3, 0.9, -1.9), scale=(1.5, 1.5, 1.5))))),
         "instances_affine": dict(scene=dict(
             objects=(dict(n_tris=400, seed=5, material="plastic", size=0.35), dict(n_tris=150, seed=9, material="glass", size=0.5),
                      dict(n_tris=300, seed=13, material="metal", size=0.3)),
             instances=(dict(object=0, center=(0.0, 0.0, -2.4), rotate=(35.0, 1.0, 2.0, -0.5)),
                        dict(object=0, center=(1.2, 0.8, -2.0), scale=(0.7, 1.4, 1.0), rotate=(60.0, 0.3, -1.0, 0.2)),
                        dict(object=2, center=(-1.2, 0.9, -1.9), scale=(1.5, 0.6, 1.2), rotate=(-50.0, 1.0, 1.0, 0.0), order="TRS"),
                        dict(object=1, center=(-1.1, -0.7, -2.2), scale=(1.0, 1.0, -1.3), rotate=(120.0, -0.4, 0.7, 1.0)),
                        dict(object=2, center=(0.9, -0.8, -2.1), scale=(1.2, 1.2, 1.2), rotate=(25.0, 0.0, 0.0, 1.0), order="RTS"),
                        dict(object=0, center=(0.3, -1.1, -1.6), scale=(-0.8, 0.9, 0.9), rotate=(80.0, 2.0, -1.0, 1.0)),
                        dict(object=1)))),
         "delta_lights": dict(scene=dict(delta_lights=(
             dict(kind="point", from_=(0.5, 1.5, -2.5), I=6.0),
             dict(kind="spot", from_=(-2.0, 2.0, -3.0), to=(0.0, 0.0, 0.0), I=(30.0, 24.0, 18.0), coneangle=25.0, conedelta=8.0),
             dict(kind="distant", from_=(1.0, 2.0, -3.0), to=(0.0, 0.0, 0.0), L=0.8)))),
         "delta_power": dict(scene=dict(delta_lights=(
             dict(kind="point", from_=(-1.0, 0.5, -2.8), I=9.0),
             dict(kind="spot", from_=(2.0, 2.5, -2.0), to=(0.2, -0.1, 0.0), I=40.0, coneangle=35.0, conedelta=35.0),
             dict(kind="distant", from_=(0.0, 1.0, -1.0), to=(0.0, 0.0, 0.0), L=(1.0, 0.9, 0.8))))),
         "analytic_point": dict(scene=dict(spheres=(dict(center=(0, 0, 0), radius=1.0, material="matte", reverse_orientation=True),),
                                           delta_lights=(dict(kind="point", from_=(0, 0, 0), I=3.14159265358979323846),)),
                                camera=dict(eye=(0, 0, 0), look=(0, 0, 1), fov=45.0)),
         "analytic_4points": dict(scene=dict(spheres=(dict(center=(0, 0, 0), radius=1.0, material="matte", reverse_orientation=True),),
                                             delta_lights=tuple(dict(kind="point", from_=(0, 0, 0), I=3.14159265358979323846 / 4)
                                                                for _ in range(4))),
                                  camera=dict(eye=(0, 0, 0), look=(0, 0, 1), fov=45.0, sampler="halton")),
         "analytic_area": dict(scene=dict(spheres=(dict(center=(0, 0, 0), radius=1.0, material="matte", reverse_orientation=True,
                                                        emit=0.5),)),
                               camera=dict(eye=(0, 0, 0), look=(0, 0, 1), fov=45.0)),
         "filter_gaussian": dict(camera=dict(pixel_filter="gaussian")),
         "filter_mitchell": dict(camera=dict(pixel_filter="mitchell", max_sample_luminance=20.0)),
         "filter_sinc": dict(camera=dict(pixel_filter="sinc", sampler="halton")),
         "filter_aniso_crop": dict(camera=dict(pixel_filter="gaussian_aniso", crop_window=(0.21, 0.83, 0.1, 0.74))),
         "filter_triangle": dict(camera=dict(pixel_filter="triangle", lens_radius=0.05, focal_distance=4.5)),
         "filter_box1": dict(camera=dict(pixel_filter="box1")),
         "sphere_light": dict(scene=dict(spheres=(dict(center=(0.5, 2.5, -2.0), radius=0.3, emit=400.0),
                                                  dict(center=(-0.6, 0.2, -2.0), radius=0.5, material="plastic"))),
                              camera=dict(sampler="halton")),
         "sphere_power": dict(scene=dict(spheres=(dict(center=(0.0, 0.0, -2.4), radius=0.25, emit=150.0, two_sided=True),
                                                  dict(center=(2.2, -1.0, 0.0), radius=0.6, emit=30.0,
                                                       reverse_orientation=True),
                                                  dict(center=(-0.7, 0.5, -1.9), radius=0.35, material="glass_rough"))))}

# VolPathIntegrator (integrators/volpath.cpp) renders of the reference, groundwork for media (SURVEY 8(f) row 4, last item):
# golden name -> (base case above, homogeneous medium around the whole scene or None, light sample strategy)
VOLPATH = {
    "volpath_four": ("four", None, "uniform"),  # no medium: still differs from "path" (light sampling at specular vertices)
    "volpath_fog": ("four", dict(sigma_a=(0.05, 0.08, 0.12), sigma_s=(0.3, 0.25, 0.2), g=0.4), "uniform"),
    "volpath_fog_delta": ("delta_lights", dict(sigma_a=(0.02, 0.02, 0.02), sigma_s=(0.5, 0.5, 0.5), g=-0.3), "spatial"),
    "volpath_fog_spheres": ("spheres", dict(sigma_a=(0.1, 0.05, 0.02), sigma_s=(0.15, 0.2, 0.3), g=0.0), "power"),
}

# Media bounded by surfaces (oracle groundwork: the device does not support them yet): null-material spheres around a
# homogeneous medium -- golden name -> (medium around the scene or None, sphere specs); 3000-triangle "four" scene
_CLOUD = dict(sigma_a=(0.3, 0.2, 0.1), sigma_s=(2.0, 2.5, 3.0), g=0.5)
VOLPATH_BOUNDED = {
    "volpath_cloud": (None, (dict(center=(0.1, 0.0, -2.2), radius=0.7, boundary=_CLOUD),)),
    "volpath_cloud_fog": (dict(sigma_a=(0.02, 0.02, 0.02), sigma_s=(0.1, 0.1, 0.1), g=0.2),
                          (dict(center=(0.1, 0.0, -2.2), radius=0.7, boundary=_CLOUD),
                           dict(center=(-1.0, 0.6, -1.8), radius=0.4, boundary=dict(sigma_a=(1, 1, 1), sigma_s=(0.5, 0.5, 0.5), g=-0.2)),
                           dict(center=(1.2, 1.8, -1.5), radius=0.35, emit=60.0))),
}
