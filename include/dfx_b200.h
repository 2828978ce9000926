/* dfx_b200.h — C-ABI of the H100-native DiligentFX PostProcess chain.
 *
 * This is the drop-in boundary (SURVEY.md §8b): every entry point is `extern "C"`, takes plain pointers /
 * sizes / POD structs, never throws and returns a dfx_status. It replaces, for the PostProcess hot path only,
 * what the reference records through DiligentCore's IDeviceContext inside
 *   PostFXContext::Execute                 (PostProcess/Common/src/PostFXContext.cpp:287-338)
 *   ScreenSpaceAmbientOcclusion::Execute   (PostProcess/ScreenSpaceAmbientOcclusion/src/ScreenSpaceAmbientOcclusion.cpp:348-387)
 *   ScreenSpaceReflection::Execute         (PostProcess/ScreenSpaceReflection/src/ScreenSpaceReflection.cpp:300-341)
 *   Bloom::Execute                         (PostProcess/Bloom/src/Bloom.cpp:407-436)
 *   TemporalAntiAliasing::Execute          (PostProcess/TemporalAntiAliasing/src/TemporalAntiAliasing.cpp:169-201)
 *   ToneMap()                              (Shaders/PostProcess/ToneMapping/public/ToneMapping.fxh:87-226)
 *
 * Two layers:
 *   1. pass level   `dfx_pass_*`  — one stateless call per reference render pass (or fused pass group); every
 *                                   plane is passed explicitly. This is what the parity tests drive.
 *   2. effect level `dfx_<effect>_{create,prepare,execute,get_plane,destroy}` — owns the effect's internal
 *                                   planes (history ping-pong, pyramids) exactly like the reference classes own
 *                                   their textures; the C++ headers under include/dfx/ wrap these in C++ classes with the
 *                                   reference's own signatures.
 *
 * All device pointers are CUDA device pointers on the current device; `stream` is a cudaStream_t passed as void*.
 * There is no CPU fallback: every entry fails with DFX_ERR_CUDA when no sm_90 device/driver is usable.
 */
#ifndef DFX_B200_H
#define DFX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFX_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------------------ */
/* status                                                                                                       */
typedef enum dfx_status
{
    DFX_OK               = 0,
    DFX_ERR_INVALID_ARG  = 1, /* null pointer, bad format, mismatched size (reference: DEV_CHECK_ERR)        */
    DFX_ERR_CUDA         = 2, /* a CUDA runtime call or launch failed; see dfx_last_error()                   */
    DFX_ERR_NOT_PREPARED = 3, /* execute before prepare (reference: TemporalAntiAliasing.cpp:178-183)         */
    DFX_ERR_UNSUPPORTED  = 4  /* unknown feature-flag bits, or a combination this build has no kernel for   */
} dfx_status;

DFX_API const char* dfx_last_error(void);           /* thread-local message of the last non-OK status      */
DFX_API int         dfx_version(void);              /* 10000*major + 100*minor + patch                     */
DFX_API uint64_t    dfx_launch_count(void);         /* kernels launched by this library so far (process)   */

/* ------------------------------------------------------------------------------------------------------------ */
/* planes                                                                                                       */
typedef enum dfx_format
{
    DFX_FORMAT_UNKNOWN = 0,
    DFX_FORMAT_R32F    = 1, /* depth, AO, history length, variance, roughness …            4 B/texel */
    DFX_FORMAT_RG32F   = 2, /* motion vectors, blue noise                                  8 B/texel */
    DFX_FORMAT_RGBA32F = 3, /* colour, normal (xyz_), material, radiance, bloom levels    16 B/texel */
    DFX_FORMAT_R8U     = 4, /* SSR reflection mask (stands in for the D16 stencil mask)    1 B/texel */
    /* transfer formats (dfx_pass_unpack_plane / dfx_pass_pack_ldr8 only; the passes compute on the fp32 formats above) */
    DFX_FORMAT_RGBA16F = 5, /* scene colour, normal as the G-buffer stores them             8 B/texel */
    DFX_FORMAT_RG16F   = 6, /* motion vectors                                               4 B/texel */
    DFX_FORMAT_RG8U    = 7, /* material (roughness, metallic) UNORM                         2 B/texel */
    DFX_FORMAT_RGBA8U  = 8, /* tone-mapped sRGB frame as a swap chain stores it             4 B/texel */
    /* shadow-map formats (dfx_shadow_convert_to_filterable only; every other entry refuses them) */
    DFX_FORMAT_R16U    = 9, /* D16_UNORM depth: code k reads as k / 65535                  2 B/texel */
    DFX_FORMAT_RG16U   = 10 /* RG16_UNORM variance shadow map: code k reads as k / 65535   4 B/texel */
} dfx_format;

/* A pitched 2-D array in HBM: row y starts at (char*)ptr + y*pitch_bytes. Stands in for ITextureView. */
typedef struct dfx_plane
{
    void*    ptr;
    size_t   pitch_bytes;
    int32_t  width;
    int32_t  height;
    int32_t  format; /* dfx_format */
    int32_t  flags;  /* DFX_PLANE_FLAG_*; 0 for every plane but a reversed depth buffer */
} dfx_plane;
/* A DEPTH plane (or level 0 of a depth pyramid) that stores reversed depth: near = 1, far = 0. Stands in for
 * PostFXContext::FEATURE_FLAG_REVERSED_DEPTH (PostFXContext.hpp:54) at the pass level, where the reference compiles the
 * POSTFX/SSAO/SSR_OPTION_INVERTED_DEPTH shader variants (ComputeClosestMotion.fx:5-9,36-40; SSAO_Common.fxh:6-23;
 * SSR_Common.fxh:6-12,48-55; SSR_ComputeIntersection.fx:109-124): the passes that read the plane take the closest depth
 * as the maximum, the far plane as 0 and the background test as depth < 1e-6. The effect-level objects set it themselves
 * from the PostFX feature flag.                                                                                  */
#define DFX_PLANE_FLAG_REVERSED_DEPTH 1
/* A depth plane (level 0 of the SSAO prefiltered-depth pyramid) that the reference would keep in R16_UNORM
 * (ScreenSpaceAmbientOcclusion::FEATURE_FLAG_HALF_PRECISION_DEPTH, …cpp:96-97). The plane stays fp32 here — this library
 * models none of the reference's narrow storage formats — but the AO pass uses the larger self-occlusion offset the
 * reference compiles in for that mode (0.005 instead of 0.00001, SSAO_ComputeAmbientOcclusion.fx:145-150).          */
#define DFX_PLANE_FLAG_HALF_PRECISION_DEPTH 2

#define DFX_MAX_MIPS 8
/* A mip chain of planes (level i is max(w>>i,1) x max(h>>i,1)). Stands in for a mip-mapped ITexture. */
typedef struct dfx_pyramid
{
    dfx_plane level[DFX_MAX_MIPS];
    int32_t   levels;
    int32_t   reserved;
} dfx_pyramid;

/* Row range [y0, y1) of the full frame that a call computes. {0, height} = whole frame. Used by the row-strip
 * multi-GPU path (SURVEY.md §8e): every GPU holds full-size planes and computes only its strip; halo rows are
 * exchanged between calls. For pyramid passes y0/y1 must be multiples of 64 (or y1 == height).               */
typedef struct dfx_rows
{
    int32_t y0;
    int32_t y1;
} dfx_rows;

/* ------------------------------------------------------------------------------------------------------------ */
/* constant blocks — byte-identical to the reference's shared C++/HLSL structs                                  */

typedef struct dfx_float4x4 { float m[4][4]; } dfx_float4x4; /* row-major, row-vector convention mul(v, M) */

/* == HLSL::CameraAttribs, Shaders/Common/public/BasicStructures.fxh:84-149 (576 bytes) */
typedef struct dfx_camera_attribs
{
    float f4Position[4];
    float f4ViewportSize[4]; /* (width, height, 1/width, 1/height) */
    float fNearPlaneZ, fFarPlaneZ, fNearPlaneDepth, fFarPlaneDepth;
    float fSceneNearZ, fSceneFarZ, fSceneNearDepth, fSceneFarDepth;
    float    fHandness;
    uint32_t uiFrameIndex;
    float    Padding0, Padding1;
    float fFocusDistance, fFStop, fFocalLength, fSensorWidth;
    float fSensorHeight, fExposure;
    float f2Jitter[2];
    dfx_float4x4 mView, mProj, mViewProj, mViewInv, mProjInv, mViewProjInv;
    float f4ExtraData[5][4];
} dfx_camera_attribs;

/* == HLSL::ScreenSpaceAmbientOcclusionAttribs, …/ScreenSpaceAmbientOcclusionStructures.fxh:64-98 (48 bytes) */
typedef struct dfx_ssao_attribs
{
    float    EffectRadius;                /* 1.0   */
    float    EffectFalloffRange;          /* 0.615 */
    float    RadiusMultiplier;            /* 1.457 */
    float    DepthMIPSamplingOffset;      /* 3.3   */
    float    TemporalStabilityFactor;     /* 0.9   */
    float    SpatialReconstructionRadius; /* 4.0   */
    int32_t  ResetAccumulation;           /* FALSE */
    float    AlphaInterpolation;          /* 1.0   */
    float    BitmaskThickness;            /* 0.5   */
    uint32_t Algorithm;                   /* DFX_SSAO_ALGORITHM_GTAO */
    float    Padding0, Padding1;
} dfx_ssao_attribs;
#define DFX_SSAO_ALGORITHM_GTAO 0
#define DFX_SSAO_ALGORITHM_HBAO 1
#define DFX_SSAO_ALGORITHM_VBAO 2

/* == HLSL::ScreenSpaceReflectionAttribs, …/ScreenSpaceReflectionStructures.fxh:43-80 (48 bytes) */
typedef struct dfx_ssr_attribs
{
    float    DepthBufferThickness;               /* 0.025 */
    float    RoughnessThreshold;                 /* 0.2   */
    uint32_t MostDetailedMip;                    /* 0     */
    int32_t  IsRoughnessPerceptual;              /* TRUE  */
    uint32_t RoughnessChannel;                   /* 0     */
    uint32_t MaxTraversalIntersections;          /* 128   */
    float    GGXImportanceSampleBias;            /* 0.3   */
    float    SpatialReconstructionRadius;        /* 4.0   */
    float    TemporalRadianceStabilityFactor;    /* 1.0   */
    float    TemporalVarianceStabilityFactor;    /* 0.9   */
    float    BilateralCleanupSpatialSigmaFactor; /* 0.9   */
    float    AlphaInterpolation;                 /* 1.0   */
} dfx_ssr_attribs;

/* == HLSL::BloomAttribs, …/BloomStructures.fxh:12-34 (32 bytes) */
typedef struct dfx_bloom_attribs
{
    float Intensity;          /* 0.15  */
    float Threshold;          /* 1.0   */
    float SoftTreshold;       /* 0.125 */
    float Radius;             /* 0.75  */
    float AlphaInterpolation; /* 1.0   */
    float Padding0, Padding1, Padding2;
} dfx_bloom_attribs;

/* == HLSL::TemporalAntiAliasingAttribs, …/TemporalAntiAliasingStructures.fxh:35-46 (16 bytes) */
typedef struct dfx_taa_attribs
{
    float   TemporalStabilityFactor; /* 0.9375 */
    int32_t ResetAccumulation;       /* FALSE  */
    int32_t SkipRejection;           /* FALSE  */
    float   Padding0;
} dfx_taa_attribs;

/* == HLSL::DepthOfFieldAttribs, Shaders/PostProcess/DepthOfField/public/DepthOfFieldStructures.fxh:31-56 (32 bytes) */
typedef struct dfx_dof_attribs
{
    float   MaxCircleOfConfusion;    /* 0.01   : largest CoC in texture coordinates                    */
    float   TemporalStabilityFactor; /* 0.9375                                                         */
    int32_t BokehKernelRingCount;    /* 5      : rings of the Octaweb kernel (2..5)                    */
    int32_t BokehKernelRingDensity;  /* 7      : samples per ring step (2..7)                          */
    float   AlphaInterpolation;      /* 1.0                                                            */
    float   Padding0, Padding1, Padding2;
} dfx_dof_attribs;
#define DFX_DOF_FEATURE_FLAG_NONE                      0u
#define DFX_DOF_FEATURE_FLAG_ENABLE_TEMPORAL_SMOOTHING (1u << 0) /* D2 (DepthOfField.hpp:65) */
#define DFX_DOF_FEATURE_FLAG_ENABLE_KARIS_INVERSE      (1u << 1) /* HDR-weighted gather in D8 (:67) */

/* == HLSL::ToneMappingAttribs (+AgXAttribs), …/ToneMappingStructures.fxh:24-52 (48 bytes) */
typedef struct dfx_tonemap_attribs
{
    int32_t  iToneMappingMode;     /* DFX_TONE_MAPPING_MODE_UNCHARTED2 */
    int32_t  bAutoExposure;        /* TRUE  */
    float    fMiddleGray;          /* 0.18  */
    int32_t  bLightAdaptation;     /* TRUE  */
    float    fWhitePoint;          /* 3.0   */
    float    fLuminanceSaturation; /* 1.0   */
    uint32_t Padding0, Padding1;
    float    AgXSaturation, AgXSlope, AgXPower, AgXOffset; /* 1,1,1,0 */
} dfx_tonemap_attribs;
#define DFX_TONE_MAPPING_MODE_NONE          0
#define DFX_TONE_MAPPING_MODE_EXP           1
#define DFX_TONE_MAPPING_MODE_REINHARD      2
#define DFX_TONE_MAPPING_MODE_REINHARD_MOD  3
#define DFX_TONE_MAPPING_MODE_UNCHARTED2    4
#define DFX_TONE_MAPPING_MODE_FILMIC_ALU    5
#define DFX_TONE_MAPPING_MODE_LOGARITHMIC   6
#define DFX_TONE_MAPPING_MODE_ADAPTIVE_LOG  7
#define DFX_TONE_MAPPING_MODE_AGX           8
#define DFX_TONE_MAPPING_MODE_AGX_CUSTOM    9
#define DFX_TONE_MAPPING_MODE_PBR_NEUTRAL  10
#define DFX_TONE_MAPPING_MODE_COMMERCE     11

/* == HLSL::CoordinateGridAttribs, Shaders/Common/public/CoordinateGridStructures.fxh:6-29 (192 bytes) */
typedef struct dfx_coordinate_grid_attribs
{
    float PositiveXAxisColor[4]; /* (1, 0, 0, 1)          */
    float PositiveYAxisColor[4]; /* (0, 1, 0, 1)          */
    float PositiveZAxisColor[4]; /* (0, 0, 1, 1)          */
    float NegativeXAxisColor[4]; /* (0.40, 0.15, 0.15, 1) */
    float NegativeYAxisColor[4]; /* (0.15, 0.40, 0.15, 1) */
    float NegativeZAxisColor[4]; /* (0.15, 0.15, 0.40, 1) */
    float XAxisWidth, YAxisWidth, ZAxisWidth; /* 3, 3, 3 pixels */
    float Padding0;
    float GridMajorColor[4];     /* (0.4, 0.4, 0.4, 1)    */
    float GridMinorColor[4];     /* (0.1, 0.1, 0.1, 1)    */
    float GridScale[4];          /* (1, 1, 1, 0): YZ, XZ, XY */
    float GridSubdivision[4];    /* (10, 10, 10, 0)       */
    float GridLineWidth;         /* 2 pixels              */
    float GridMinCellWidth;      /* 4 pixels              */
    float GridMinCellSize;       /* 0.0001                */
    float Padding1;
} dfx_coordinate_grid_attribs;
/* CoordinateGridRenderer::FEATURE_FLAGS (Components/interface/CoordinateGridRenderer.hpp:59-84) */
#define DFX_GRID_FEATURE_FLAG_NONE            0u
#define DFX_GRID_FEATURE_FLAG_CONVERT_TO_SRGB (1u << 0)
#define DFX_GRID_FEATURE_FLAG_RENDER_PLANE_YZ (1u << 1)
#define DFX_GRID_FEATURE_FLAG_RENDER_PLANE_XZ (1u << 2)
#define DFX_GRID_FEATURE_FLAG_RENDER_PLANE_XY (1u << 3)
#define DFX_GRID_FEATURE_FLAG_RENDER_AXIS_X   (1u << 4)
#define DFX_GRID_FEATURE_FLAG_RENDER_AXIS_Y   (1u << 5)
#define DFX_GRID_FEATURE_FLAG_RENDER_AXIS_Z   (1u << 6)
#define DFX_GRID_FEATURE_FLAG_ALL             127u

/* Selection highlighting: HnPostProcessTaskParams' selection fields (Hydrogent/interface/Tasks/HnPostProcessTask.hpp:79-85), the
 * background depth of HnPostProcessTask (:220) and the selected prim (HnProcessSelectionTask.cpp:293-301). 48 bytes. */
typedef struct dfx_selection_attribs
{
    float    SelectionColor[4];              /* (1, 0.675, 0.25, 0.5)                                          */
    float    OccludedSelectionColor[4];      /* (0.375, 0.375, 0.125, 0.5)                                     */
    float    SelectionOutlineWidth;          /* 4 pixels; also the jump flood's MaximumDistance (HnTaskManager.cpp:698-700) */
    float    NonselectionDesaturationFactor; /* 0                                                              */
    float    ClearDepth;                     /* the background depth: 1 (0 with reversed depth)                */
    uint32_t selection_id;                   /* stands in for SelectedPrimId: a change resets TAA's history    */
} dfx_selection_attribs;

/* == cbEnvMapRenderAttribs, Shaders/Common/private/EnvMap.psh:11-21 (80 bytes): what EnvMapRenderer::Prepare writes
 * (Components/src/EnvMapRenderer.cpp:226-242), Scale = float4(RenderAttribs::Scale, 1). */
typedef struct dfx_env_map_attribs
{
    dfx_tonemap_attribs ToneMapping;   /* the ToneMappingAttribs argument of Prepare            */
    float               AverageLogLum; /* 1 (RenderAttribs default): ToneMap's argument as is  */
    float               MipLevel;      /* 0                                                    */
    float               Alpha;         /* 1: the alpha written with the colour                 */
    float               Padding0;
    float               Scale[4];      /* (1, 1, 1, 1): multiplies the sampled rgb             */
} dfx_env_map_attribs;
/* EnvMapRenderer::PSOKey::ENV_MAP_TYPE (Components/interface/EnvMapRenderer.hpp): a cube map or a sphere map */
#define DFX_ENV_MAP_TYPE_CUBE   0
#define DFX_ENV_MAP_TYPE_SPHERE 1
/* EnvMapRenderer::OPTION_FLAGS (Components/interface/EnvMapRenderer.hpp) */
#define DFX_ENV_MAP_OPTION_NONE                   0u
#define DFX_ENV_MAP_OPTION_CONVERT_OUTPUT_TO_SRGB (1u << 0)
#define DFX_ENV_MAP_OPTION_COMPUTE_MOTION_VECTORS (1u << 1)
#define DFX_ENV_MAP_OPTION_USE_REVERSE_DEPTH      (1u << 2)
#define DFX_ENV_MAP_OPTION_ALL                    7u

/* == BoundBoxAttribs, Shaders/Common/private/BoundBoxStructures.fxh (96 bytes): what BoundBoxRenderer::Prepare writes
 * (Components/src/BoundBoxRenderer.cpp:224-255). Transform is the matrix as the shader reads it: a box corner c in [0, 1]^3 goes to
 * mul(float4(c, 1), Transform) (row vector times matrix, row-major here). */
typedef struct dfx_bound_box_attribs
{
    dfx_float4x4 Transform;     /* identity: the unit cube                                                    */
    float        Color[4];      /* (1, 1, 1, 1): stored as given                                             */
    float        PatternLength; /* 32: pixels                                                                 */
    uint32_t     PatternMask;   /* 0xFFFFFFFF: bit k fills the k-th 1/32 of the pattern                       */
    float        Padding0;
    float        Padding1;
} dfx_bound_box_attribs;
/* BoundBoxRenderer::OPTION_FLAGS (Components/interface/BoundBoxRenderer.hpp) */
#define DFX_BOUND_BOX_OPTION_NONE                   0u
#define DFX_BOUND_BOX_OPTION_CONVERT_OUTPUT_TO_SRGB (1u << 0)
#define DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS (1u << 1)
#define DFX_BOUND_BOX_OPTION_USE_REVERSE_DEPTH      (1u << 2)
#define DFX_BOUND_BOX_OPTION_ALL                    7u

/* VectorFieldRenderer::RenderAttribs' values (Components/interface/VectorFieldRenderer.hpp), what Render (VectorFieldRenderer.cpp:173-223)
 * writes into VectorField.vsh's constant block: ScaleAndBias = (Scale, Bias), the grid size as float and as uint, the two colours. */
typedef struct dfx_vector_field_attribs
{
    float    Bias[2];       /* (0, 0): added to the field's value first                         */
    float    Scale[2];      /* (1, 1): then multiplied, in NDC units                              */
    float    StartColor[4]; /* (1, 1, 1, 1): the colour at the cell's centre                      */
    float    EndColor[4];   /* (1, 1, 1, 1): the colour at the vector's end                       */
    uint32_t GridSize[2];   /* (0, 0): lines across and down; 0 in either draws nothing           */
} dfx_vector_field_attribs;
/* VectorFieldRenderer::RenderAttribs::ConvertOutputToSRGB */
#define DFX_VECTOR_FIELD_OPTION_NONE                   0u
#define DFX_VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB (1u << 0)
#define DFX_VECTOR_FIELD_OPTION_ALL                    1u

/* Default-initialisers (the reference's DEFAULT_VALUE()s). */
DFX_API void dfx_ssao_attribs_default(dfx_ssao_attribs* a);
DFX_API void dfx_ssr_attribs_default(dfx_ssr_attribs* a);
DFX_API void dfx_bloom_attribs_default(dfx_bloom_attribs* a);
DFX_API void dfx_dof_attribs_default(dfx_dof_attribs* a);
DFX_API void dfx_taa_attribs_default(dfx_taa_attribs* a);
DFX_API void dfx_tonemap_attribs_default(dfx_tonemap_attribs* a);
DFX_API void dfx_coordinate_grid_attribs_default(dfx_coordinate_grid_attribs* a);
DFX_API void dfx_selection_attribs_default(dfx_selection_attribs* a);
/* EnvMapRenderer::RenderAttribs' defaults (AverageLogLum 1, MipLevel 0, Alpha 1, Scale (1, 1, 1)) with dfx_tonemap_attribs_default */
DFX_API void dfx_env_map_attribs_default(dfx_env_map_attribs* a);
/* BoundBoxRenderer::RenderAttribs' defaults: the identity transform, Color (1, 1, 1, 1), PatternLength 32, PatternMask 0xFFFFFFFF */
DFX_API void dfx_bound_box_attribs_default(dfx_bound_box_attribs* a);
/* VectorFieldRenderer::RenderAttribs' defaults: Bias (0, 0), Scale (1, 1), both colours (1, 1, 1, 1), GridSize (0, 0) */
DFX_API void dfx_vector_field_attribs_default(dfx_vector_field_attribs* a);
/* The attribs HnPostProcessTask draws the motion-vector view with (Hydrogent/src/Tasks/HnPostProcessTask.cpp:932-938) over a
 * width x height final target: GridSize (width / 20, height / 20), Scale -0.02 / max(elapsed_time, 0.001) in both axes (the vectors
 * point against the motion), StartColor (1, 1, 1, 1), EndColor (0.5, 0.5, 0.5, 1), Bias 0. */
DFX_API void dfx_vector_field_attribs_hydrogent(uint32_t width, uint32_t height, float elapsed_time, dfx_vector_field_attribs* a);

/* == PostFXContext::FrameDesc, PostProcess/Common/interface/PostFXContext.hpp:68-84 */
typedef struct dfx_frame_desc
{
    uint32_t Index;
    uint32_t Width;
    uint32_t Height;
    uint32_t OutputWidth;
    uint32_t OutputHeight;
} dfx_frame_desc;

/* feature flags: numeric values of the reference enums */
#define DFX_POSTFX_FEATURE_FLAG_NONE                 0u
#define DFX_POSTFX_FEATURE_FLAG_REVERSED_DEPTH       (1u << 0) /* depth: near = 1, far = 0 (see DFX_PLANE_FLAG_REVERSED_DEPTH) */
#define DFX_POSTFX_FEATURE_FLAG_HALF_PRECISION_DEPTH (1u << 1) /* accepted; selects a storage format only, planes stay fp32 */
#define DFX_POSTFX_FEATURE_FLAG_TEMPORAL_UPSCALING   (1u << 2) /* Bloom runs at FrameDesc.OutputWidth x OutputHeight (Bloom.cpp:84-85) */
#define DFX_SSAO_FEATURE_FLAG_NONE                   0u
#define DFX_SSAO_FEATURE_FLAG_HALF_PRECISION_DEPTH   (1u << 0) /* AO self-occlusion offset 0.005; planes stay fp32 */
#define DFX_SSAO_FEATURE_FLAG_HALF_RESOLUTION        (1u << 1) /* A0 + A1-A3 at width/2 x height/2 + A4 */
#define DFX_SSR_FEATURE_FLAG_NONE                    0u
#define DFX_SSR_FEATURE_FLAG_PREVIOUS_FRAME          (1u << 0)
#define DFX_SSR_FEATURE_FLAG_HALF_RESOLUTION         (1u << 1) /* S3 + S4 at width/2 x height/2 */
#define DFX_BLOOM_FEATURE_FLAG_NONE                  0u
#define DFX_TAA_FEATURE_FLAG_NONE                    0u
#define DFX_TAA_FEATURE_FLAG_GAUSSIAN_WEIGHTING      (1u << 0)
#define DFX_TAA_FEATURE_FLAG_BICUBIC_FILTER          (1u << 1)
#define DFX_TAA_FEATURE_FLAG_YCOCG_COLOR_SPACE       (1u << 2)

/* ============================================================================================================ */
/* 1. pass level                                                                                                */
/* ============================================================================================================ */

/* P0 ComputeBlueNoiseTexture (PostFXContext.cpp:567-609; Shaders/Common/private/ComputeBlueNoiseTexture.fx:81-89).
 * tables: device pointer to the 131,328-byte blob (Sobol_256d[256] ++ ScramblingTile[128*128*8]).
 * xy, zw: 128x128 RG32F.                                                                                       */
DFX_API dfx_status dfx_pass_blue_noise(void* stream, const uint8_t* tables, uint32_t frame_index,
                                       const dfx_plane* xy, const dfx_plane* zw);

/* P1+P2+P3 fused: ComputeReprojectedDepth (ComputeReprojectedDepth.fx:18-30), ComputeClosestMotion
 * (ComputeClosestMotion.fx:24-55), ComputePreviousDepth (PostFXContext.cpp:657-676).
 * cameras: device pointer to dfx_camera_attribs[2] = {curr, prev}.                                             */
DFX_API dfx_status dfx_pass_postfx_prepare(void* stream, const dfx_camera_attribs* cameras_dev,
                                           const dfx_plane* curr_depth, const dfx_plane* prev_depth_in,
                                           const dfx_plane* motion,
                                           const dfx_plane* reprojected_depth, const dfx_plane* closest_motion,
                                           const dfx_plane* previous_depth, dfx_rows rows);

/* A1+A2 ComputePrefilteredDepth (ScreenSpaceAmbientOcclusion.cpp:843-957; SSAO_ComputePrefilteredDepthBuffer.fx:79-122).
 * pyr->level[0] aliases the input depth (the reference's CopyTextureDepth into mip 0 is elided); levels 1..4 written. */
DFX_API dfx_status dfx_pass_ssao_prefilter_depth(void* stream, const dfx_camera_attribs* cameras_dev,
                                                 const dfx_ssao_attribs* attribs, const dfx_pyramid* pyr, dfx_rows rows);

/* FEATURE_FLAG_HALF_RESOLUTION (ScreenSpaceAmbientOcclusion.hpp:59-82): A0 builds a width/2 x height/2 checkerboard of the 2x2
 * min / max depth, A1-A3 run on it (the prefiltered pyramid, hence the occlusion target, is half size: A3 recognises the
 * mode by a pyramid of half the normal plane's size and doubles GetInvViewportSize(), SSAO_ComputeAmbientOcclusion.fx:68-75),
 * and A4 brings the occlusion back to full resolution for A5-A8.
 * A0 ComputeDepthCheckerboard (…cpp:818-841; SSAO_ComputeDownsampledDepth.fx:8-29). `rows`: rows of the half-size plane. */
DFX_API dfx_status dfx_pass_ssao_downsample_depth(void* stream, const dfx_plane* depth, const dfx_plane* out_half, dfx_rows rows);
/* A4 ComputeBilateralUpsampling (…cpp:992-1020; SSAO_ComputeBilateralUpsampling.fx:62-139): 3x3 joint-bilateral filter of
 * the half-size occlusion guided by the full-resolution depth; background pixels get 1.0.                        */
DFX_API dfx_status dfx_pass_ssao_upsample(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* depth,
                                          const dfx_plane* occlusion_half, const dfx_plane* out_occlusion, dfx_rows rows);

/* A3 ComputeAmbientOcclusion (…cpp:961-990; SSAO_ComputeAmbientOcclusion.fx:132-231). Includes the clear to 1.0. */
DFX_API dfx_status dfx_pass_ssao_ambient_occlusion(void* stream, const dfx_camera_attribs* cameras_dev,
                                                   const dfx_ssao_attribs* attribs, const dfx_pyramid* prefiltered_depth,
                                                   const dfx_plane* normal, const dfx_plane* blue_noise_zw,
                                                   const dfx_plane* occlusion, dfx_rows rows);

/* A5 ComputeTemporalAccumulation (…cpp:1032-1073; SSAO_ComputeTemporalAccumulation.fx:151-182). Includes the
 * clears of both targets to 1.0 (background pixels keep 1.0).                                                  */
DFX_API dfx_status dfx_pass_ssao_temporal(void* stream, const dfx_camera_attribs* cameras_dev,
                                          const dfx_ssao_attribs* attribs,
                                          const dfx_plane* curr_occlusion, const dfx_plane* prev_occlusion,
                                          const dfx_plane* prev_history_length, const dfx_plane* reprojected_depth,
                                          const dfx_plane* previous_depth, const dfx_plane* closest_motion,
                                          const dfx_plane* out_occlusion, const dfx_plane* out_history_length,
                                          dfx_rows rows);

/* A6 ComputeConvolutedDepthHistory (…cpp:1075-1255; SSAO_ComputeConvolutedDepthHistory.fx:93-109).
 * level[0] of both pyramids are inputs (accumulated AO, depth); levels 1..4 written.                           */
DFX_API dfx_status dfx_pass_ssao_convolute(void* stream, const dfx_pyramid* occlusion_pyr, const dfx_pyramid* depth_pyr,
                                           dfx_rows rows);

/* A7 ComputeResampledHistory (…cpp:1257-1286; SSAO_ComputeResampledHistory.fx:56-115). */
DFX_API dfx_status dfx_pass_ssao_resample(void* stream, const dfx_camera_attribs* cameras_dev,
                                          const dfx_pyramid* occlusion_pyr, const dfx_pyramid* depth_pyr,
                                          const dfx_plane* history_length, const dfx_plane* normal,
                                          const dfx_plane* out_occlusion, dfx_rows rows);

/* A8 ComputeSpatialReconstruction (…cpp:1288-1329; SSAO_ComputeSpatialReconstruction.fx:49-100). The reference's
 * CopyTexture(resolved -> history[curr]) is elided: `out_occlusion` IS history[curr].                          */
DFX_API dfx_status dfx_pass_ssao_spatial(void* stream, const dfx_camera_attribs* cameras_dev,
                                         const dfx_ssao_attribs* attribs,
                                         const dfx_plane* occlusion, const dfx_plane* history_length,
                                         const dfx_plane* depth, const dfx_plane* normal,
                                         const dfx_plane* out_occlusion, dfx_rows rows);

/* S1 ComputeHierarchicalDepthBuffer (ScreenSpaceReflection.cpp:777-902; SSR_ComputeHierarchicalDepthBuffer.fx:30-73).
 * level[0] aliases the input depth; levels 1..6 written.                                                       */
DFX_API dfx_status dfx_pass_ssr_hiz(void* stream, const dfx_pyramid* pyr, dfx_rows rows);

/* S2 ComputeStencilMaskAndExtractRoughness (…cpp:904-932; SSR_ComputeStencilMaskAndExtractRoughness.fx:13-40).
 * mask (R8U): 1 where the pixel is a reflection sample, 0 elsewhere; roughness written only where mask==1.     */
DFX_API dfx_status dfx_pass_ssr_mask_roughness(void* stream, const dfx_ssr_attribs* attribs,
                                               const dfx_plane* material, const dfx_plane* depth,
                                               const dfx_plane* roughness, const dfx_plane* mask, dfx_rows rows);

/* The front of a frame in one pass over the depth plane: P1+P2+P3 (dfx_pass_postfx_prepare), S1 (dfx_pass_ssr_hiz, levels 1..6 of
 * `hiz`), S2 (dfx_pass_ssr_mask_roughness) and A2 (dfx_pass_ssao_prefilter_depth, levels 1..4 of `prefiltered`), whole frame.
 * Every output is bit-identical to those four passes (with the pyramids built one launch per level). One kernel stages a TMA tile of
 * depth per 64x64 block and writes the per-pixel outputs and the pyramid levels up to min(trailing zero bits of the frame size, 4);
 * the levels above go through the pyramid passes' own kernels. When that kernel cannot run (fewer than 2 such levels, a depth plane
 * TMA cannot describe: base or pitch not 16-byte aligned) the four passes run instead. level[0] of both pyramids is not read:
 * curr_depth is level 0. cameras: device pointer to dfx_camera_attribs[2] = {curr, prev}.                                   */
DFX_API dfx_status dfx_pass_front_prepare(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_ssr_attribs* ssr_attribs,
                                          const dfx_ssao_attribs* ssao_attribs, const dfx_plane* curr_depth, const dfx_plane* prev_depth_in,
                                          const dfx_plane* motion, const dfx_plane* material, const dfx_plane* reprojected_depth,
                                          const dfx_plane* closest_motion, const dfx_plane* previous_depth, const dfx_plane* roughness,
                                          const dfx_plane* mask, const dfx_pyramid* hiz, const dfx_pyramid* prefiltered);

/* FEATURE_FLAG_HALF_RESOLUTION (ScreenSpaceReflection.hpp:64-76): S3 downsamples the mask, S4 traces one ray per 2x2 block
 * into width/2 x height/2 targets (which of the four pixels: a 4x4 pattern, PostFX_Common.fxh:45-55), S5 gathers from the
 * half-size targets; S6 / S7 are unchanged. S4 and S5 recognise the mode by intersect planes of half the frame size.
 * S3 ComputeDownsampledStencilMask (…cpp:934-961; SSR_ComputeDownsampledStencilMask.fx:13-61): 1 where the closest depth
 * and the largest roughness of the 2x2 (+ odd row / column) footprint pass IsReflectionSample. `rows`: of the half-size mask. */
DFX_API dfx_status dfx_pass_ssr_downsample_mask(void* stream, const dfx_ssr_attribs* attribs, const dfx_plane* roughness,
                                                const dfx_plane* depth, const dfx_plane* mask_half, dfx_rows rows);

/* S4 ComputeIntersection (…cpp:963-999; SSR_ComputeIntersection.fx:281-325). Includes both clears to 0.
 * motion may be NULL unless DFX_SSR_FEATURE_FLAG_PREVIOUS_FRAME is set in `flags`.                             */
DFX_API dfx_status dfx_pass_ssr_intersect(void* stream, const dfx_camera_attribs* cameras_dev,
                                          const dfx_ssr_attribs* attribs, uint32_t flags,
                                          const dfx_plane* color, const dfx_plane* normal, const dfx_plane* roughness,
                                          const dfx_plane* mask, const dfx_plane* blue_noise_xy,
                                          const dfx_pyramid* hiz, const dfx_plane* motion,
                                          const dfx_plane* out_radiance, const dfx_plane* out_raydir_pdf, dfx_rows rows);

/* S4 for one frame split into row strips over several GPUs of an NVLink / NVSwitch box (SURVEY.md §8e). The march of a ray may
 * cross the whole screen. The Hi-Z pyramid `hiz` (depth included) must be COMPLETE on this GPU - the march walks it in a dependent
 * chain of ~36 loads per ray, which must not cross the link (measured; the strips executor all-gathers it by peer stores) - while
 * the colour and the normal at the hit, two independent loads per ray, are loaded straight from the GPU that OWNS the row (peer
 * loads; every GPU holds full-size RGBA32F planes at the same pitch, valid on its own rows only). `color`, `normal` describe the
 * local planes; `peers` gives, per rank, the base pointer of the same plane as mapped into this process (cudaIpcOpenMemHandle, or a
 * plain pointer when one process drives all GPUs; base[own rank] = the local pointer; the `hiz` entries are not used).
 * row_begin[r] .. row_begin[r+1] are the rows rank r owns; every boundary but the last is a multiple of 64. Output is bit-identical
 * to dfx_pass_ssr_intersect on complete planes. DFX_SSR_FEATURE_FLAG_PREVIOUS_FRAME is not supported. The caller orders the
 * producers on all GPUs before this launch (stream-ordered barrier) and this launch before the next frame's writers. No reference
 * counterpart: the reference renders a frame on one device.                                                        */
#define DFX_MAX_PEERS 8
typedef struct dfx_peer_set {
    int32_t     count;                                  /* GPUs sharing the frame, 1..DFX_MAX_PEERS                    */
    int32_t     row_begin[DFX_MAX_PEERS + 1];
    const void* color[DFX_MAX_PEERS];
    const void* normal[DFX_MAX_PEERS];
    const void* hiz[DFX_MAX_MIPS][DFX_MAX_PEERS];       /* level 0 = the depth plane                                   */
} dfx_peer_set;
/* The same frame-sharding description in the form the strips executor (section 4) uses: every rank holds ALL planes at the same
 * offsets of an identically laid-out slab; base[r] is rank r's slab as mapped into this process (dfx_ipc_open), so the copy of any
 * plane on rank r is at (plane pointer - base[rank] + base[r]). Rows are owned in 64-row blocks: rank r owns [row_begin[r], row_begin[r+1]). */
typedef struct dfx_peer_map {
    int32_t     count, rank;
    int32_t     row_begin[DFX_MAX_PEERS + 1];
    const void* base[DFX_MAX_PEERS];
} dfx_peer_map;
DFX_API dfx_status dfx_pass_ssr_intersect_peer(void* stream, const dfx_camera_attribs* cameras_dev,
                                               const dfx_ssr_attribs* attribs, uint32_t flags, const dfx_peer_set* peers,
                                               const dfx_plane* color, const dfx_plane* normal, const dfx_plane* roughness,
                                               const dfx_plane* mask, const dfx_plane* blue_noise_xy, const dfx_pyramid* hiz,
                                               const dfx_plane* out_radiance, const dfx_plane* out_raydir_pdf, dfx_rows rows);
/* cudaDeviceEnablePeerAccess(peer_device) for the current device; OK if already enabled, DFX_ERR_UNSUPPORTED if the
 * two devices have no peer path.                                                                                   */
DFX_API dfx_status dfx_enable_peer_access(int32_t peer_device);
/* Device memory another process on the same box can map (one process per GPU): dfx_ipc_alloc = cudaMalloc +
 * cudaIpcGetMemHandle on the current device; the 64-byte handle travels over any host channel; dfx_ipc_open maps it into
 * the CURRENT device's address space (cudaIpcMemLazyEnablePeerAccess), so kernels of the opening process may load from
 * it over NVLink. The owner keeps the allocation alive until every peer has called dfx_ipc_close.                  */
#define DFX_IPC_HANDLE_BYTES 64
DFX_API dfx_status dfx_ipc_alloc(size_t bytes, void** out_ptr, uint8_t handle[DFX_IPC_HANDLE_BYTES]);
DFX_API dfx_status dfx_ipc_free(void* ptr);
DFX_API dfx_status dfx_ipc_open(const uint8_t handle[DFX_IPC_HANDLE_BYTES], void** out_ptr);
DFX_API dfx_status dfx_ipc_close(void* mapped);

/* S5 ComputeSpatialReconstruction (…cpp:1001-1031; SSR_ComputeSpatialReconstruction.fx:114-172). Masked writes. */
DFX_API dfx_status dfx_pass_ssr_spatial(void* stream, const dfx_camera_attribs* cameras_dev,
                                        const dfx_ssr_attribs* attribs,
                                        const dfx_plane* roughness, const dfx_plane* mask, const dfx_plane* normal,
                                        const dfx_plane* depth, const dfx_plane* raydir_pdf, const dfx_plane* radiance,
                                        const dfx_plane* out_resolved_radiance, const dfx_plane* out_resolved_variance,
                                        const dfx_plane* out_resolved_depth, dfx_rows rows);

/* S6 ComputeTemporalAccumulation (…cpp:1033-1069; SSR_ComputeTemporalAccumulation.fx:224-263). Masked writes. */
DFX_API dfx_status dfx_pass_ssr_temporal(void* stream, const dfx_camera_attribs* cameras_dev,
                                         const dfx_ssr_attribs* attribs, const dfx_plane* mask,
                                         const dfx_plane* motion, const dfx_plane* hit_depth,
                                         const dfx_plane* reprojected_depth, const dfx_plane* curr_radiance,
                                         const dfx_plane* curr_variance, const dfx_plane* previous_depth,
                                         const dfx_plane* prev_radiance, const dfx_plane* prev_variance,
                                         const dfx_plane* out_radiance, const dfx_plane* out_variance, dfx_rows rows);

/* S6 on a row strip of a frame sharded over several GPUs: the previous-frame planes (previous depth, radiance and variance history),
 * which the pass reads at reprojected positions that no fixed halo bounds, are loaded from the GPU that owns the row. The three planes
 * must lie in the caller's slab (peers->base[peers->rank]). Bit-identical to dfx_pass_ssr_temporal on complete planes. */
DFX_API dfx_status dfx_pass_ssr_temporal_peer(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_ssr_attribs* attribs,
                                              const dfx_peer_map* peers, const dfx_plane* mask, const dfx_plane* motion,
                                              const dfx_plane* hit_depth, const dfx_plane* reprojected_depth,
                                              const dfx_plane* curr_radiance, const dfx_plane* curr_variance,
                                              const dfx_plane* previous_depth, const dfx_plane* prev_radiance,
                                              const dfx_plane* prev_variance, const dfx_plane* out_radiance,
                                              const dfx_plane* out_variance, dfx_rows rows);

/* S7 ComputeBilateralCleanup (…cpp:1071-1104; SSR_ComputeBilateralCleanup.fx:49-97). Includes the clear to 0. */
DFX_API dfx_status dfx_pass_ssr_bilateral(void* stream, const dfx_camera_attribs* cameras_dev,
                                          const dfx_ssr_attribs* attribs, const dfx_plane* mask,
                                          const dfx_plane* depth, const dfx_plane* normal, const dfx_plane* roughness,
                                          const dfx_plane* radiance, const dfx_plane* variance,
                                          const dfx_plane* out, dfx_rows rows);

/* Bloom passes: `rows` is a row range of the OUTPUT plane of the call (the pyramid level being written), not of the
 * full-resolution frame — the levels have their own heights.
 * B1 ComputePrefilteredTexture (Bloom.cpp:288-311; Bloom_ComputePrefilteredTexture.fx:37-83). */
DFX_API dfx_status dfx_pass_bloom_prefilter(void* stream, const dfx_bloom_attribs* attribs,
                                            const dfx_plane* color, const dfx_plane* out_level0, dfx_rows rows);
/* B2 ComputeDownsampledTexture (Bloom.cpp:313-337; Bloom_ComputeDownsampledTexture.fx:11-41). */
DFX_API dfx_status dfx_pass_bloom_downsample(void* stream, const dfx_plane* in, const dfx_plane* out, dfx_rows rows);
/* B3 ComputeUpsampledTexture, uInstID==0 (Bloom.cpp:339-375; Bloom_ComputeUpsampledTexture.fx:20-54). */
DFX_API dfx_status dfx_pass_bloom_upsample(void* stream, const dfx_plane* same_level_down, const dfx_plane* coarser,
                                           const dfx_plane* out, dfx_rows rows);
/* B4 final composite, uInstID!=0 (Bloom.cpp:373-393; Bloom_ComputeUpsampledTexture.fx:45-48). */
DFX_API dfx_status dfx_pass_bloom_composite(void* stream, const dfx_bloom_attribs* attribs,
                                            const dfx_plane* color, const dfx_plane* up0, const dfx_plane* out, dfx_rows rows);

/* B2 for the levels first .. mips-1 followed by B3 for the levels mips-2 .. first-1, in ONE launch of one thread-block cluster
 * (the reference issues one draw per level, Bloom.cpp:324-337 and :355-375; on the small levels of the pyramid those dependent
 * launches cost more than the work). `down` / `up` are arrays of `mips` planes (level i = max(level0 >> i, 1)); reads
 * down[first-1], writes down[first..mips-1] and up[first-1..mips-2]. Results are bit-identical to the per-level passes.
 * dfx_bloom_tail_first_level: the level the effect object hands over to this pass (`mips` = none). Off by default (dfx_tune "bloom_tail" =
 * 1 switches it on: first level with <= "bloom_tail_texels" = 2048 texels): as a pass the cluster launch beats the per-level launches of the
 * same levels, but a cluster occupies 8 SMs of one GPC while it walks the levels, and under async compute the whole frame is faster
 * without it. */
#define DFX_BLOOM_MAX_LEVELS 16
DFX_API dfx_status dfx_pass_bloom_tail(void* stream, const dfx_plane* down, const dfx_plane* up, int32_t first, int32_t mips);
DFX_API int32_t    dfx_bloom_tail_first_level(const dfx_plane* down, int32_t mips);
/* The same contract as dfx_pass_bloom_tail for levels of ANY size, in one cooperative launch over the whole GPU: a level is a phase
 * of a persistent grid, phases are separated by a grid-wide barrier (replaces the 5 + 5 draws of Bloom.cpp:324-337 / :355-375 at 4K).
 * `workspace`: 64 bytes of device memory, 16-byte aligned, zeroed once by the caller and used by one launch at a time (the kernel
 * leaves it zeroed). A barrier that is not reached within ~2 s raises an error word in the workspace instead of hanging the GPU:
 * dfx_bloom_levels_check reads it back (synchronises). Same taps in the same order as the per-level passes (results agree to the last
 * bit or two: FMA contraction). The effect object uses it when dfx_tune "bloom_levels" is 1; default 0 - under async compute the per-level
 * launches overlap the next frame better than a grid that needs the whole GPU. */
DFX_API dfx_status dfx_pass_bloom_levels(void* stream, const dfx_plane* down, const dfx_plane* up, int32_t first, int32_t mips, void* workspace);
DFX_API dfx_status dfx_bloom_levels_check(const void* workspace, int32_t* timed_out);

/* T1 ComputeTemporalAccumulation (TemporalAntiAliasing.cpp:260-289; TAA_ComputeTemporalAccumulation.fx:229-261). */
DFX_API dfx_status dfx_pass_taa(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_taa_attribs* attribs,
                                uint32_t flags, const dfx_plane* curr_color, const dfx_plane* prev_accum,
                                const dfx_plane* closest_motion, const dfx_plane* reprojected_depth,
                                const dfx_plane* previous_depth, const dfx_plane* out_accum, dfx_rows rows);

/* Compose step between SSAO and TAA, reduced form (SURVEY.md §8f rank 1; Hydrogent/shaders/HnPostProcess.psh:145-185):
 *   rgb += ssr.rgb * ssr.a * ssr_scale;  rgb *= lerp(1, ao, ssao_scale);  alpha passes through.
 * ssr / ao may be NULL (scale treated as 0).                                                                   */
DFX_API dfx_status dfx_pass_compose(void* stream, const dfx_plane* color, const dfx_plane* ssr, const dfx_plane* ao,
                                    float ssr_scale, float ssao_scale, const dfx_plane* out, dfx_rows rows);

/* DepthOfField (PostProcess/DepthOfField/src/DepthOfField.cpp:292-331; Shaders/PostProcess/DepthOfField/private/DOF_*.fx), the
 * eleven passes in execution order. `rows` is always a row range of the OUTPUT plane of the call. Sizes: CoC planes
 * W x H; dilation level k (W >> k) x (H >> k), k = 0..3; prefiltered / bokeh planes (W/2) x (H/2), alpha = CoC of the layer.
 *   D1  coc            signed circle of confusion in [-1, 1] from depth and the lens fields of the camera (…CircleOfConfusion.fx:24-39)
 *   D2  temporal_coc   history reprojected by the closest motion, clamped to mean +- 2.5 sigma (…TemporalCircleOfConfusion.fx:54-92)
 *   D3  separated_coc  near field |CoC| (CoC < 0) -> dilation level 0 (…SeparatedCircleOfConfusion.fx:5-11)
 *   D4  dilation       2x2 (+ odd row / column) maximum, called for levels 1..3 (…DilationCircleOfConfusion.fx:16-52)
 *   D5/6 blur_coc      13-tap Gaussian (radius 6, sigma 5), horizontal into an intermediate plane, vertical back (…BlurredCoC.fx:8-28)
 *   D7  prefilter      SDR-weighted 2x2 mean -> foreground (alpha: blurred dilation, linear) and background (alpha: max far CoC)
 *   D8  bokeh, first   gather over the Octaweb kernel (rings, density from attribs), optional HDR ("Karis inverse") weights
 *   D9  bokeh, second  flood fill with the small 3 x 5 kernel (component-wise maximum)
 *   D10 postfilter     2x2 tent
 *   D11 combine        far layer, then near layer over the full-resolution colour by smoothstep(0.1, 1, alpha)            */
DFX_API dfx_status dfx_pass_dof_coc(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_dof_attribs* attribs,
                                    const dfx_plane* depth, const dfx_plane* out_coc, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_temporal_coc(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_dof_attribs* attribs,
                                             const dfx_plane* curr_coc, const dfx_plane* prev_coc, const dfx_plane* closest_motion,
                                             const dfx_plane* out_coc, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_separated_coc(void* stream, const dfx_plane* coc, const dfx_plane* out, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_dilation(void* stream, const dfx_plane* last, const dfx_plane* out, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_blur_coc(void* stream, const dfx_plane* coc, int32_t vertical, const dfx_plane* out, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_prefilter(void* stream, const dfx_plane* color, const dfx_plane* coc, const dfx_plane* dilation,
                                          const dfx_plane* out_fg, const dfx_plane* out_bg, dfx_rows rows);
/* radiance (the full-resolution colour) is read only with DFX_DOF_FEATURE_FLAG_ENABLE_KARIS_INVERSE in `flags`; may be NULL otherwise */
DFX_API dfx_status dfx_pass_dof_bokeh(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_dof_attribs* attribs, uint32_t flags,
                                      int32_t second_pass, const dfx_plane* fg, const dfx_plane* bg, const dfx_plane* radiance,
                                      const dfx_plane* out_fg, const dfx_plane* out_bg, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_postfilter(void* stream, const dfx_plane* fg, const dfx_plane* bg, const dfx_plane* out_fg,
                                           const dfx_plane* out_bg, dfx_rows rows);
DFX_API dfx_status dfx_pass_dof_combine(void* stream, const dfx_dof_attribs* attribs, const dfx_plane* color, const dfx_plane* dof_near,
                                        const dfx_plane* dof_far, const dfx_plane* out, dfx_rows rows);

/* Compose step, full form (Hydrogent/shaders/HnPostProcess.psh:145-185; host HnPostProcessTask.cpp:834-869). With
 * Opacity = color.a:
 *   rgb += (GetSpecularIBL_GGX(surface, view, ssr.rgb) - specular_ibl.rgb) * ssr.a * ssr_scale * Opacity
 *   rgb *= lerp(1, ao, ssao_scale * Opacity);                       alpha passes through
 * i.e. the reflection is re-weighted by the split-sum BRDF of the surface (metallic-roughness workflow, PBR_Shading.fxh:
 * 220-302 with USE_IBL_MULTIPLE_SCATTERING = 1, :429-451; material.x = roughness, material.y = metallic) and exchanged for
 * the image-based specular term the renderer had already added. `brdf_lut` = dfx_pass_precompute_brdf_lut (RG32F, sampled
 * linear-clamp at (N.V, roughness)). ssr == NULL skips the first line (the five planes it needs may then be NULL too);
 * ao == NULL skips the second.                                                                                     */
DFX_API dfx_status dfx_pass_compose_ibl(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* color,
                                        const dfx_plane* ssr, const dfx_plane* ao, const dfx_plane* specular_ibl,
                                        const dfx_plane* normal, const dfx_plane* base_color, const dfx_plane* material,
                                        const dfx_plane* brdf_lut, float ssr_scale, float ssao_scale, const dfx_plane* out,
                                        dfx_rows rows);
/* Pre-integrated GGX table (Shaders/PBR/private/PrecomputeBRDF.psh:10-48; PBR_Renderer.cpp:548-625 builds it once at
 * 512 x 512 with 512 samples): texel (x, y) = (scale, bias) of the split sum at N.V = (x + .5)/w, roughness = (y + .5)/h. */
DFX_API dfx_status dfx_pass_precompute_brdf_lut(void* stream, uint32_t num_samples, const dfx_plane* out_lut);

/* M1+M2 ToneMap() (ToneMapping.fxh:87-226) + optional LinearToSRGB (SRGBUtilities.fxh:27-33), as used by
 * Hydrogent/shaders/HnCopyFrame.psh:32-62. ave_log_lum is the already exposure-scaled fAveLogLum argument.     */
DFX_API dfx_status dfx_pass_tonemap(void* stream, const dfx_tonemap_attribs* attribs, float ave_log_lum,
                                    int32_t convert_to_srgb, const dfx_plane* color, const dfx_plane* out, dfx_rows rows);

/* Fused variants (an element-wise pass is evaluated inside the kernel that consumes / produces its plane, so the
 * intermediate frame never makes a round trip through HBM). Same arithmetic per pixel as the separate passes.
 *   compose + T1 : `color` is the un-composed scene colour; the composed colour is computed on the fly.
 *   B4 + M1/M2   : writes the tone-mapped LDR frame directly; only for exact 2:1 levels and an even rows.y0
 *                  (DFX_ERR_UNSUPPORTED otherwise). */
DFX_API dfx_status dfx_pass_compose_taa(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_taa_attribs* attribs, uint32_t flags,
                                        const dfx_plane* color, const dfx_plane* ssr, const dfx_plane* ao, float ssr_scale, float ssao_scale,
                                        const dfx_plane* prev_accum, const dfx_plane* closest_motion, const dfx_plane* reprojected_depth,
                                        const dfx_plane* previous_depth, const dfx_plane* out_accum, dfx_rows rows);
DFX_API dfx_status dfx_pass_bloom_composite_tonemap(void* stream, const dfx_bloom_attribs* attribs, const dfx_tonemap_attribs* tonemap, float ave_log_lum,
                                                    int32_t convert_to_srgb, const dfx_plane* color, const dfx_plane* up0, const dfx_plane* ldr_out,
                                                    dfx_rows rows);

/* G1 coordinate grid and axes (Components/src/CoordinateGridRenderer.cpp:233-287 RenderGridAxes; Shaders/Common/private/
 * CoordinateGridPS.psh:24-38; Shaders/Common/public/CoordinateGrid.fxh:158-227): per pixel, the grid of the planes and the axes
 * that `flags` (DFX_GRID_FEATURE_FLAG_*) select, evaluated at the pixel's depth with MinDepth = MaxDepth, optionally converted to
 * sRGB (FEATURE_FLAG_CONVERT_TO_SRGB), then alpha-blended into `color_inout` in place (BS_AlphaBlend, DESIGN.md §2:
 * rgb = src.rgb * src.a + dst.rgb * (1 - src.a), a = src.a + dst.a * (1 - src.a)). cameras_dev[0] = the camera (device memory);
 * `attribs` is a host pointer. depth R32F, color_inout RGBA32F, same size. Flags without a plane or axis bit draw nothing and
 * leave the plane untouched (no launch).                                                                                        */
DFX_API dfx_status dfx_pass_coordinate_grid(void* stream, const dfx_camera_attribs* cameras_dev, uint32_t flags,
                                            const dfx_coordinate_grid_attribs* attribs, const dfx_plane* depth,
                                            const dfx_plane* color_inout, dfx_rows rows);
/* G2 the final copy-frame step with the grid (Hydrogent/shaders/HnCopyFrame.psh:27-63 with ENABLE_GRID; host
 * HnPostProcessTask.cpp:380-495): ToneMap (the same operator code as dfx_pass_tonemap; ave_log_lum is the already exposure-scaled
 * argument), then the grid of `grid_flags` evaluated over the 3x3 depth min / max around the pixel (out-of-frame texels read 0),
 * `rgb = lerp(rgb, grid.rgb, grid.a)`, then LinearToSRGB when convert_to_srgb. Alpha passes through. The grid's own
 * CONVERT_TO_SRGB bit has no effect here, as in the shader. color RGBA32F (what Bloom, DepthOfField or TAA produced), depth R32F
 * (the frame's current depth, HnPostProcessTask.cpp:471), out RGBA32F. grid_flags == 0 is refused: that is dfx_pass_tonemap.  */
DFX_API dfx_status dfx_pass_copy_frame_grid(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_tonemap_attribs* tonemap,
                                            float ave_log_lum, int32_t convert_to_srgb, uint32_t grid_flags,
                                            const dfx_coordinate_grid_attribs* grid_attribs, const dfx_plane* color,
                                            const dfx_plane* depth, const dfx_plane* out, dfx_rows rows);

/* E the environment-map background (Components/src/EnvMapRenderer.cpp:102-190 GetPSO, :244-252 Render; Shaders/Common/private/
 * EnvMap.vsh, EnvMap.psh:45-73 SampleEnvMap), in place on the G-buffer's colour and motion planes. A full-screen triangle at
 * z = fFarPlaneDepth of cameras_dev[0] with the depth test LESS_EQUAL (GREATER_EQUAL with DFX_ENV_MAP_OPTION_USE_REVERSE_DEPTH) and
 * depth writes off (:175-176): a pixel is drawn when fFarPlaneDepth <= depth (>= reversed); any other pixel (NaN depth included)
 * is not written at all. A drawn pixel, with ClipPos = (NDC x, NDC y, fFarPlaneDepth, 1) at the pixel centre (DESIGN.md §2):
 *   WorldPos = ClipPos * mViewProjInv, Direction = WorldPos.xyz / WorldPos.w - f4Position.xyz;
 *   rgb = SampleLevel(env_map, normalize(Direction), MipLevel).rgb * Scale.rgb, the sampler Sam_LinearClamp (trilinear, the LOD
 *     clamped to the map's levels; the cube filtered across its faces by the rule of DESIGN.md §2; the sphere at
 *     TransformDirectionToSphereMapUV(dir), ShaderUtilities.fxh:98-102);
 *   ToneMap(rgb, ToneMapping, AverageLogLum) when ToneMapping.iToneMappingMode != NONE (no exposure factor);
 *   pow(rgb, 1 / 2.2) with DFX_ENV_MAP_OPTION_CONVERT_OUTPUT_TO_SRGB (not LinearToSRGB);
 *   colour = (rgb, Alpha);
 *   with DFX_ENV_MAP_OPTION_COMPUTE_MOTION_VECTORS: motion = GetMotionVector(ClipPos.xy, PrevClipPos.xy, Jitter, PrevJitter) with
 *     PrevClipPos = float4(cameras_dev[1].f4Position.xyz + Direction, 1) * mViewProj of cameras_dev[1], xy / w (the motion of a point
 *     at infinity: it depends on the rotation only).
 * This stands in for the pipeline's RenderTargetMask: the colour is always written, the motion only with motion vectors on (then
 * motion_inout is required; without, it may be NULL and is not touched). `type` DFX_ENV_MAP_TYPE_*: a cube is a pyramid whose level i
 * is one plane of s_i x 6*s_i texels (width x height), faces stacked top to bottom in the order +X, -X, +Y, -Y, +Z, -Z; a sphere is
 * an ordinary pyramid. Level i of either is max(w0 >> i, 1) x max(h0 >> i, 1) (a cube: s_i = max(s0 >> i, 1)). Map texels RGBA32F or
 * RGBA16F; depth R32F; color_inout RGBA32F or RGBA16F; motion_inout RG32F or RG16F; the 16-bit stores round to nearest even. Any
 * row range; only its rows are touched. Refuses an unknown type, option bit or tone-mapping mode, a cube level that is not s x 6s,
 * a mip chain of other sizes, mismatched plane sizes and motion vectors without a motion plane. */
DFX_API dfx_status dfx_pass_env_map(void* stream, const dfx_camera_attribs* cameras_dev, int32_t type, const dfx_pyramid* env_map,
                                    uint32_t options, const dfx_env_map_attribs* attribs, const dfx_plane* depth,
                                    const dfx_plane* color_inout, const dfx_plane* motion_inout, dfx_rows rows);

/* The most levels an IBL source map or output chain may have (a 32768^2 map's full chain; a 2048^2 HDRI has 12). */
#define DFX_MAX_ENV_LEVELS 16
/* IBL cube-map precomputation (PBR/src/PBR_Renderer.cpp:729-970 PrecomputeCubemaps): the image-based-lighting cubes a PBR renderer
 * samples, convolved from an environment map. Both passes draw every texel of every face of their output with the texel direction
 * N = normalize(CubemapFace.vsh at the pixel centre: g_Rotation[face] * (x, y, 1, 1), x = 2(i + 1/2)/s - 1, y = 1 - 2(j + 1/2)/s),
 * through the face matrices of PBR_Renderer.cpp:913-922 as float values (DESIGN.md §2), and sample the source with E's sampler
 * (Sam_LinearClamp: trilinear, the seamless cube rule of DESIGN.md §2). Each sample is the reference shader's arithmetic, one rounding
 * per operation, transcendentals correctly rounded; the samples of a texel are summed in another order than the shader's, within
 * the bound DESIGN.md §2 derives.
 *   env_type   DFX_ENV_MAP_TYPE_CUBE (level i is s_i x 6 s_i, faces +X, -X, +Y, -Y, +Z, -Z stacked) or DFX_ENV_MAP_TYPE_SPHERE
 *              (a lat-long map w_i x h_i); env_levels[0..n_env) its mip chain, level i max(w0 >> i, 1) x max(h0 >> i, 1) (cube:
 *              s_i = max(s0 >> i, 1)), 1 <= n_env <= DFX_MAX_ENV_LEVELS, RGBA32F or RGBA16F, one format for all levels. g_EnvMipCount
 *              is n_env; g_EnvMapWidth / Height are level 0's face size (cube) or w0 x h0 (sphere).
 *   num_samples 0 = the reference default: 8192 for the irradiance (GetDefaultDiffuseSamplesCount on a discrete adapter), 256 for
 *              the prefilter.
 *   optimize_samples  OPTIMIZE_SAMPLES: 1 picks each sample's LOD from its solid angle (mip bias 1), 0 reads level 0.
 *   outputs    cube planes s x 6s, RGBA16F (IrradianceCubeFmt / PrefilteredEnvMapFmt) or RGBA32F, stored rounded to nearest even.
 * Nothing else is read or written; the work is enqueued on `stream` without host synchronisation.                                */
/* ComputeIrradianceMap.psh: rgb = the mean of SampleLevel(L_k) over the cosine-weighted directions L_k around N, alpha 1. */
DFX_API dfx_status dfx_pass_irradiance_cube(void* stream, int32_t env_type, const dfx_plane* env_levels, int32_t n_env,
                                            uint32_t num_samples, int32_t optimize_samples, const dfx_plane* out);
/* PrefilterEnvMap.psh: out_levels[0..n_out) is a chain (level m is max(s0 >> m, 1) x 6 of that, one format, 2 <= n_out <=
 * DFX_MAX_ENV_LEVELS) and level m is prefiltered at PerceptualRoughness m / (n_out - 1) (PBR_Renderer.cpp:951): rgb =
 * sum(SampleLevel(L_k) * NoL_k) / sum(NoL_k) over the GGX-importance-sampled reflections L_k of R = N, alpha 0. All levels are
 * written by one launch. n_out = 1 is refused: the reference divides 0 by 0 there. */
DFX_API dfx_status dfx_pass_prefilter_env_map(void* stream, int32_t env_type, const dfx_plane* env_levels, int32_t n_env,
                                              uint32_t num_samples, int32_t optimize_samples, const dfx_plane* out_levels, int32_t n_out);

/* Shadow modes (BasicStructures.fxh SHADOW_MODE_*) and the most cascades a shadow map has (MAX_CASCADES). */
#define DFX_SHADOW_MODE_PCF   1
#define DFX_SHADOW_MODE_VSM   2
#define DFX_SHADOW_MODE_EVSM2 3
#define DFX_SHADOW_MODE_EVSM4 4
#define DFX_MAX_CASCADES      8
/* CascadeAttribs (BasicStructures.fxh:6-14), 64 bytes. */
typedef struct dfx_cascade_attribs
{
    float f4LightSpaceScale[4];
    float f4LightSpaceScaledBias[4];
    float f4StartEndZ[4];
    float f4MarginProjSpace[4]; /* the cascade margin in light projection space */
} dfx_cascade_attribs;
/* ShadowMapAttribs (BasicStructures.fxh:28-67, the C++ form), 1200 bytes; BOOL fields are 32-bit. The defaults are the struct's
 * DEFAULT_VALUEs (capi.ShadowMapAttribs.default()). ConvertToFilterable reads iNumCascades, Cascades[i].f4LightSpaceScale.xy,
 * fEVSMPositiveExponent, fEVSMNegativeExponent, bIs32BitEVSM, iFixedFilterSize and fFilterWorldSize. */
typedef struct dfx_shadow_map_attribs
{
    dfx_float4x4        mWorldToLightView;
    dfx_cascade_attribs Cascades[DFX_MAX_CASCADES];
    dfx_float4x4        mWorldToShadowMapUVDepth[DFX_MAX_CASCADES];
    float               fCascadeCamSpaceZEnd[DFX_MAX_CASCADES];
    float               f4ShadowMapDim[4]; /* Width, Height, 1/Width, 1/Height */
    int32_t iNumCascades;                  /* 0 */
    float   fNumCascades;                  /* 0 */
    int32_t bVisualizeCascades;            /* 0 */
    int32_t bVisualizeShadowing;           /* 0 */
    float   fReceiverPlaneDepthBiasClamp;  /* 10 */
    float   fFixedDepthBias;               /* 1e-5 */
    float   fCascadeTransitionRegion;      /* 0.1 */
    int32_t iMaxAnisotropy;                /* 4 */
    float   fVSMBias;                      /* 1e-4 */
    float   fVSMLightBleedingReduction;    /* 0 */
    float   fEVSMPositiveExponent;         /* 40 */
    float   fEVSMNegativeExponent;         /* 5 */
    int32_t bIs32BitEVSM;                  /* 1 */
    int32_t iFixedFilterSize;              /* 3: a 3x3 filter */
    float   fFilterWorldSize;              /* 0 */
    int32_t fDummy;
} dfx_shadow_map_attribs;
/* The filter radii ConvertToFilterable uses for cascade `cascade` of a width x height shadow map (ShadowMapManager.cpp:560-579):
 * (iFixedFilterSize - 1) / 2 on both axes when iFixedFilterSize > 0; otherwise, in float and in this order,
 * fFilterWorldSize * f4LightSpaceScale.x * 0.5f / 2.f * width and the same with .y and height. Host only. Refuses a null pointer and
 * a cascade outside 0..DFX_MAX_CASCADES-1. */
DFX_API dfx_status dfx_shadow_filter_radii(const dfx_shadow_map_attribs* attribs, int32_t cascade, int32_t width, int32_t height,
                                           float* horz_radius, float* vert_radius);
/* ShadowMapManager::ConvertToFilterable (Components/src/ShadowMapManager.cpp:533-600; Shaders/Shadows/private/ShadowConversions.fx):
 * the variance shadow maps of every cascade, from the depth the application rendered into each cascade. For cascade i, with the
 * radii of dfx_shadow_filter_radii, VSMHorzPS (VSM) or EVSMHorzPS (EVSM2, EVSM4) then VertBlurPS, bit for bit by the rules of
 * DESIGN.md §2: tap i of range = int(floor(r + 0.5)) weighs GetSampleWeight(i, r); moments are summed in tap order, one rounding per
 * operation, then divided by the summed weight; an out-of-range depth tap reads 0 (warped for EVSM), an out-of-range row of the
 * horizontal result reads 0; the horizontal result is stored in the filterable format (and read back from it) before the vertical
 * pass; EVSM's exponents are clamped to 42 (32-bit) or 5.54 (16-bit) and exp is correctly rounded. iFixedFilterSize == 2 skips the
 * vertical pass: the horizontal result is the filterable map.
 *   shadow_map   n planes, one per cascade, all w x h (at most 16384 each way) and DFX_FORMAT_R16U (D16_UNORM) or R32F (D32_FLOAT).
 *   filterable   n planes of the same size in the mode's filterable format, all the same: VSM RG16U or RG32F, EVSM2 RG16F or RG32F,
 *                EVSM4 RGBA16F or RGBA32F; the 16-bit float stores round to nearest even, the UNORM store is
 *                floor(saturate(v) * 65535 + 0.5) (NaN -> 0).
 *   intermediate one w x h plane in the filterable format, the reference's one-slice intermediate. When every cascade's range is at
 *                most 16 on both axes, one fused pass keeps the horizontal result on chip; the plane may then be NULL and is not
 *                touched. Larger ranges run the reference's two passes per cascade through it.
 * PCF returns DFX_OK and does nothing, as the reference does. Refuses an unknown mode, n outside 1..DFX_MAX_CASCADES,
 * n != attribs->iNumCascades, bIs32BitEVSM disagreeing with the filterable format's width, formats or sizes other than these, a
 * missing or mismatched intermediate where the two-pass path runs, a filterable slice (or the intermediate the two-pass path uses)
 * whose bytes overlap another plane of the call (shadow-map slices may share memory: they are only read), and a radius that is negative or not finite
 * or whose range is 2^15 or more. The work is enqueued on `stream` without host synchronisation. */
DFX_API dfx_status dfx_shadow_convert_to_filterable(void* stream, int32_t mode, const dfx_shadow_map_attribs* attribs,
                                                    const dfx_plane* shadow_map, int32_t n, const dfx_plane* filterable,
                                                    const dfx_plane* intermediate);

/* B the selected prim's bounding box (Components/src/BoundBoxRenderer.cpp:150-168 GetPSO, :257-277 Render; Shaders/Common/private/
 * BoundBox.vsh, BoundBox.psh:27-48 GetBoundBoxOutput), in place on the G-buffer's colour and motion planes. The 24 vertices of
 * BoundBoxVS (GetBoxCorner's table through attribs->Transform, then cameras_dev[0].mViewProj; PREV_CLIP_POS through cameras_dev[1]'s)
 * make 12 lines, rasterised by the aliased-line rule of DESIGN.md §2: clipped against 0 <= z <= w, snapped to 1/256 pixel in the
 * plane-sized viewport, diamond exit, attributes at the pixel centre's projection onto the snapped segment. A fragment is kept when
 * its z / w passes the depth test LESS_EQUAL (GREATER_EQUAL with DFX_BOUND_BOX_OPTION_USE_REVERSE_DEPTH; no depth write) and the
 * pattern bit min(uint(frac(Dist / PatternLength) * PatternLength), 31) of PatternMask is set (Dist: the distance in pixels to the
 * line's first vertex, from the interpolated clip positions); a pixel keeps the last kept fragment in primitive order. A kept
 * pixel's colour is attribs->Color as given, and with DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS its motion is
 * GetMotionVector(ClipPos.xy / w, PrevClipPos.xy / w, Jitter, PrevJitter); every other pixel is not touched.
 * DFX_BOUND_BOX_OPTION_CONVERT_OUTPUT_TO_SRGB changes nothing, as in the reference (BoundBox.psh never reads it). depth R32F;
 * color_inout RGBA32F or RGBA16F; motion_inout RG32F or RG16F (required with motion vectors; otherwise it may be NULL and is not
 * touched); the 16-bit stores round to nearest even. Any row range; only its rows are touched, and they are the rows of a full call.
 * Refuses unknown option bits, mismatched plane sizes, motion vectors without a motion plane, and a PatternLength that is not finite
 * and > 0. */
DFX_API dfx_status dfx_pass_bound_box(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_bound_box_attribs* attribs, uint32_t options,
                                      const dfx_plane* depth, const dfx_plane* color_inout, const dfx_plane* motion_inout, dfx_rows rows);

/* The vector field overlay (Components/src/VectorFieldRenderer.cpp:142-157 GetPSO, :173-223 Render; Shaders/Common/private/
 * VectorField.vsh; the default PS main, :76-86), drawn over color_inout. Line k = row * GridSize.x + col runs from
 * TexUVToNormalizedDeviceXY(UV), UV = ((col + 0.5) / GridSize.x, (row + 0.5) / GridSize.y), to that point plus
 * (SampleLevel(vector_field, UV).xy + Bias) * Scale (a bilinear, clamped tap), at z = 0, w = 1, and is rasterised by the aliased-line
 * rule of DESIGN.md §2 in the target-sized viewport: never clipped; a non-finite or far end (beyond the guard band) draws nothing.
 * Its colour goes from StartColor to EndColor through the rule's perspective-correct t; with
 * DFX_VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB rgb becomes pow(rgb, 1 / 2.2). No depth test and no blending: a pixel several lines
 * cover takes the last line's fragment in primitive order (the highest k); every other pixel is not touched. vector_field RG32F or
 * RG16F, any size; color_inout RGBA32F or RGBA16F (the 16-bit stores round to nearest even); scratch an R32F plane of the target's
 * size whose texels are read as 32-bit words: all zero on entry, and left all zero. Any row range; only its rows are touched, and
 * they are the rows of a full call. Two launches, no host synchronisation. Refuses unknown option bits, bad or mismatched planes and
 * a GridSize whose vertex count 2 * GridSize.x * GridSize.y does not fit in 32 bits. */
DFX_API dfx_status dfx_pass_vector_field(void* stream, const dfx_vector_field_attribs* attribs, uint32_t options, const dfx_plane* vector_field,
                                         const dfx_plane* color_inout, const dfx_plane* scratch, dfx_rows rows);

/* J the closest selected location (Hydrogent/src/Tasks/HnProcessSelectionTask.cpp:304-369): HnInitClosestSelectedLocation.psh on
 * `selection_depth` (R32F; a texel != clear_depth is selected), then dfx_selection_jfa_iterations(max_distance) steps of
 * HnUpdateClosestSelectedLocation.psh with SampleRange 2^(N-1-i). `out` (RG32F) holds what the last step writes, bit for bit:
 * (x, y * 0.5 + 0.5) of the normalised centre of the closest selected pixel, or (0, 0) for none. `scratch` (RG32F, a different
 * plane) is the ping-pong plane of the steps. Whole frame; the three planes have one size. Refuses a max_distance that is not
 * positive and finite. */
DFX_API dfx_status dfx_pass_closest_selected_location(void* stream, float clear_depth, float max_distance, const dfx_plane* selection_depth,
                                                      const dfx_plane* scratch, const dfx_plane* out);
/* O selection outline (Hydrogent/shaders/HnPostProcess.psh:211-244), in place on `color_inout` (RGBA32F; alpha passes through):
 * unselected pixels (not depth != ClearDepth && selection_depth == depth) are desaturated by NonselectionDesaturationFactor, and
 * the outline saturate(1 - distance to the closest selected location / SelectionOutlineWidth), zero on selected pixels
 * (selection_depth != ClearDepth), lerps towards SelectionColor where depth == selection_depth at that location and towards
 * OccludedSelectionColor elsewhere. The colours are taken as the shader sees them (HnPostProcessTask.cpp:840-850 reverse
 * tone-maps them first when TAA and a tone map follow). depth, selection_depth R32F, closest_location RG32F (J's output), same
 * size. Refuses a SelectionOutlineWidth that is not positive and finite. */
DFX_API dfx_status dfx_pass_selection_outline(void* stream, const dfx_selection_attribs* attribs, const dfx_plane* depth,
                                              const dfx_plane* selection_depth, const dfx_plane* closest_location,
                                              const dfx_plane* color_inout, dfx_rows rows);
/* F the final compose with TAA off (Hydrogent/shaders/HnPostProcess.psh with TONE_MAPPING_MODE, ENABLE_GRID and
 * CONVERT_OUTPUT_TO_SRGB, drawn straight into the final colour target: HnPostProcessTask.cpp:158-187, :834-869). Per pixel:
 *   1. the reduced compose of dfx_pass_compose (ssr / ao NULL = scale 0);
 *   2. ToneMap of tonemap->iToneMappingMode (NONE: none; ave_log_lum is the already exposure-scaled argument, as in
 *      dfx_pass_tonemap);
 *   3. when selection != NULL: the desaturation and outline of dfx_pass_selection_outline, with the colours exactly as given;
 *   4. when grid_flags != 0: the grid of grid_flags over the pixel's own depth (MinDepth = MaxDepth, plus the camera's jitter),
 *      rgb = lerp(rgb, grid.rgb, grid.a); the grid's own CONVERT_TO_SRGB bit has no effect;
 *   5. LinearToSRGB when convert_to_srgb.
 * Alpha passes through. color RGBA32F or RGBA16F, ssr RGBA32F, ao / depth / selection_depth R32F, closest_location RG32F (J's
 * output), out RGBA32F, all one size. depth is required with the selection or the grid, cameras_dev (device memory) and
 * grid_attribs with the grid. Any row range; only its rows are stored. Refuses unknown grid flags, an unknown tone-mapping mode
 * and a SelectionOutlineWidth that is not positive and finite. */
DFX_API dfx_status dfx_pass_compose_final(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* color, const dfx_plane* ssr,
                                          const dfx_plane* ao, float ssr_scale, float ssao_scale, const dfx_tonemap_attribs* tonemap,
                                          float ave_log_lum, int32_t convert_to_srgb, const dfx_selection_attribs* selection,
                                          const dfx_plane* depth, const dfx_plane* selection_depth, const dfx_plane* closest_location,
                                          uint32_t grid_flags, const dfx_coordinate_grid_attribs* grid_attribs, const dfx_plane* out,
                                          dfx_rows rows);

/* The viewer's view modes (HN_VIEW_MODE, Hydrogent/interface/HnTypes.hpp). SHADED and WHITE_BASE_COLOR are the ordinary frame; the
 * three debug views of HnPostProcess.psh are SCENE_DEPTH, EDGE_MAP and MESH_ID. MOTION_VECTORS is named for the refusal. */
#define DFX_VIEW_MODE_SHADED           0
#define DFX_VIEW_MODE_MOTION_VECTORS   14
#define DFX_VIEW_MODE_WHITE_BASE_COLOR 19
#define DFX_VIEW_MODE_SCENE_DEPTH      24
#define DFX_VIEW_MODE_EDGE_MAP         25
#define DFX_VIEW_MODE_MESH_ID          26
#define DFX_VIEW_MODE_COUNT            27
/* F with HnPostProcess.psh's VIEW_MODE = view_mode (SCENE_DEPTH, EDGE_MAP or MESH_ID): dfx_pass_compose_final's steps and arguments,
 * with one more step per mode:
 *   SCENE_DEPTH (:130-143), before the compose, only when loading_animation_factor == 0: the colour's red channel (the renderer's
 *     scene-depth view, drawn with scene range == camera range) becomes RelZ = r * (fFarPlaneZ - fNearPlaneZ) + fNearPlaneZ,
 *     rgb = saturate((RelZ - fSceneNearZ) / max(fSceneFarZ - fSceneNearZ, 1e-6)) with cameras_dev[0]'s scene range (which
 *     dfx_pass_depth_range can write into it);
 *   EDGE_MAP (:189-202), after the tone map: rgb = min(colour edge + depth edge, 1), the colour edge over the clamped 3x3 of `color`
 *     (zero on the background, depth == fFarPlaneDepth), the depth edge over the clamped 3x3 of DepthToCameraZ(depth);
 *   MESH_ID (:204-209), after the tone map: rgb = frac(sin(ID * 3 + k) * 43758.5453), k = 0, 1, 2, ID = mesh_id + 1; black on the
 *     background.
 * The selection, grid and sRGB steps follow unchanged; alpha passes through. cameras_dev is always required, depth with EDGE_MAP and
 * MESH_ID, mesh_id (R32F, the size of out) with MESH_ID. Any row range (EDGE_MAP reads the neighbouring rows of the whole plane).
 * Refuses what dfx_pass_compose_final refuses, and any other view mode. */
DFX_API dfx_status dfx_pass_compose_view(void* stream, const dfx_camera_attribs* cameras_dev, int32_t view_mode, float loading_animation_factor,
                                         const dfx_plane* color, const dfx_plane* ssr, const dfx_plane* ao, float ssr_scale, float ssao_scale,
                                         const dfx_tonemap_attribs* tonemap, float ave_log_lum, int32_t convert_to_srgb,
                                         const dfx_selection_attribs* selection, const dfx_plane* depth, const dfx_plane* selection_depth,
                                         const dfx_plane* closest_location, const dfx_plane* mesh_id, uint32_t grid_flags,
                                         const dfx_coordinate_grid_attribs* grid_attribs, const dfx_plane* out, dfx_rows rows);

/* == HLSL::DepthRangeI (Shaders/Common/public/ComputeDepthRangeStructs.fxh), read as floats: the layout of
 * dfx_camera_attribs::fSceneNearZ .. fSceneFarDepth (16 bytes). */
typedef struct dfx_scene_depth_range
{
    float fSceneNearZ, fSceneFarZ, fSceneNearDepth, fSceneFarDepth;
} dfx_scene_depth_range;
/* R the scene's depth range (DepthRangeCalculator::ComputeRange, DepthRangeCalculator.cpp:229-272: ClearDepthRange.csh, then
 * ComputeDepthRange.csh). `out_dev` (device memory, 4 floats laid out as dfx_scene_depth_range) is first set to the camera's range
 * (near Z = fFarPlaneZ, far Z = fNearPlaneZ, near depth = fFarPlaneDepth, far depth = fNearPlaneDepth), then every non-background
 * texel (depth != fFarPlaneDepth) of `depth` (R32F) is folded in, bit for bit as the shader does: the integer min / max of asint() of
 * the per-thread, per-row and per-16x16-group float partials of the shader's groups, and of asint(DepthToCameraZ()) of them; with
 * reversed depth (fNearPlaneDepth > fFarPlaneDepth) the near and far depth swap. For non-negative depths that is the plain min / max;
 * for negative depths and -0 the grouping decides. Always the whole plane: the shader's groups are anchored at row 0, so there is no
 * row range. Passing &cameras_dev[0].fSceneNearZ writes the range into the camera, as HnComputeDepthBoundsTask does. Two launches. */
DFX_API dfx_status dfx_pass_depth_range(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* depth, float* out_dev);

/* Host-side pieces that the reference computes on the CPU. */
/* HnProcessSelectionTask::Sync (HnProcessSelectionTask.cpp:71): the number of jump-flood steps for an outline width,
 * ceil(log2(max(max_distance, 1))) + 1. */
DFX_API uint32_t dfx_selection_jfa_iterations(float max_distance);
/* ReverseExpToneMap (Components/src/ToneMapping.cpp:43-83): the HDR colour that the exponential tone map takes close to `color`. */
DFX_API void dfx_reverse_exp_tone_map(const float color[3], float middle_gray, float average_log_lum, float out[3]);
/* TemporalAntiAliasing::GetJitterOffset (TemporalAntiAliasing.cpp:63-78, Halton(2,3) x16). */
DFX_API void dfx_taa_jitter_offset(uint32_t frame_index, uint32_t width, uint32_t height, float out_jitter[2]);
/* Bloom::ComputeMipCount (Bloom.cpp:152-156) applied to the half-resolution level-0 size. */
DFX_API int32_t dfx_bloom_mip_count(uint32_t width, uint32_t height, float radius);

/* Implementation switches for A/B measurements (tools/, bench.py --tune): every value of a knob computes the same pass, through a
 * different kernel. Unknown names read as `fallback`. Also settable at load time: DFX_TUNE="name=value,name=value". */
DFX_API void    dfx_tune_set(const char* name, int32_t value);
DFX_API int32_t dfx_tune_get(const char* name, int32_t fallback);
DFX_API void    dfx_tune_unset(const char* name); /* back to the built-in default (NULL: every knob) */

/* ============================================================================================================ */
/* 2. effect level                                                                                              */
/* ============================================================================================================ */

typedef struct dfx_postfx dfx_postfx;
typedef struct dfx_ssao   dfx_ssao;
typedef struct dfx_ssr    dfx_ssr;
typedef struct dfx_bloom  dfx_bloom;
typedef struct dfx_taa    dfx_taa;

/* plane ids for dfx_*_get_plane */
enum
{
    DFX_POSTFX_PLANE_BLUE_NOISE_XY     = 0,
    DFX_POSTFX_PLANE_BLUE_NOISE_ZW     = 1,
    DFX_POSTFX_PLANE_REPROJECTED_DEPTH = 2,
    DFX_POSTFX_PLANE_PREVIOUS_DEPTH    = 3,
    DFX_POSTFX_PLANE_CLOSEST_MOTION    = 4
};
enum
{
    DFX_SSAO_PLANE_OUTPUT            = 0,  /* == GetAmbientOcclusionSRV()                       */
    DFX_SSAO_PLANE_OCCLUSION         = 1,  /* raw AO (A3)                                       */
    DFX_SSAO_PLANE_ACCUMULATED       = 2,  /* A5 output == convoluted-AO mip 0                  */
    DFX_SSAO_PLANE_HISTORY_LENGTH    = 3,  /* A5 history length of the current frame            */
    DFX_SSAO_PLANE_RESAMPLED         = 4,  /* A7                                                */
    DFX_SSAO_PLANE_UPSAMPLED         = 5,  /* A4 (half resolution only); OCCLUSION is then width/2 x height/2 */
    DFX_SSAO_PLANE_PREFILTERED_MIP0  = 10, /* +i : prefiltered depth mip i (0..4)               */
    DFX_SSAO_PLANE_CONV_AO_MIP0      = 20, /* +i : convoluted AO mip i (0..4)                   */
    DFX_SSAO_PLANE_CONV_DEPTH_MIP0   = 30  /* +i : convoluted depth mip i (0..4)                */
};
enum
{
    DFX_SSR_PLANE_OUTPUT            = 0,  /* == GetSSRRadianceSRV()                             */
    DFX_SSR_PLANE_ROUGHNESS         = 1,
    DFX_SSR_PLANE_MASK              = 2,
    DFX_SSR_PLANE_RADIANCE          = 3,
    DFX_SSR_PLANE_RAYDIR_PDF        = 4,
    DFX_SSR_PLANE_RESOLVED_RADIANCE = 5,
    DFX_SSR_PLANE_RESOLVED_VARIANCE = 6,
    DFX_SSR_PLANE_RESOLVED_DEPTH    = 7,
    DFX_SSR_PLANE_RADIANCE_HISTORY  = 8,  /* current frame's slot                               */
    DFX_SSR_PLANE_VARIANCE_HISTORY  = 9,
    DFX_SSR_PLANE_HIZ_MIP0          = 10, /* +i : Hi-Z mip i (0..6)                             */
    DFX_SSR_PLANE_MASK_HALF         = 20  /* S3 (half resolution only); RADIANCE / RAYDIR_PDF are then half size */
};
enum
{
    DFX_BLOOM_PLANE_OUTPUT    = 0,   /* == GetBloomTextureSRV()                                 */
    DFX_BLOOM_PLANE_DOWN0     = 10,  /* +i : downsampled level i                                */
    DFX_BLOOM_PLANE_UP0       = 30   /* +i : upsampled level i                                  */
};
enum
{
    DFX_TAA_PLANE_ACCUMULATED_CURR = 0, /* == GetAccumulatedFrameSRV(false)                     */
    DFX_TAA_PLANE_ACCUMULATED_PREV = 1  /* == GetAccumulatedFrameSRV(true)                      */
};

/* ---- PostFXContext (PostProcess/Common/interface/PostFXContext.hpp:51-172) ---- */
typedef struct dfx_postfx_render_attribs
{
    void*                     stream;          /* stands in for pDeviceContext                   */
    const dfx_plane*          curr_depth;      /* pCurrDepthBufferSRV  R32F                      */
    const dfx_plane*          prev_depth;      /* pPrevDepthBufferSRV  R32F                      */
    const dfx_plane*          motion_vectors;  /* pMotionVectorsSRV    RG32F                     */
    const dfx_camera_attribs* curr_camera;     /* host pointers, uploaded like PostFXContext.cpp:302-319 */
    const dfx_camera_attribs* prev_camera;
} dfx_postfx_render_attribs;

DFX_API dfx_status dfx_postfx_create(dfx_postfx** out);
DFX_API void       dfx_postfx_destroy(dfx_postfx* ctx);
DFX_API dfx_status dfx_postfx_prepare(dfx_postfx* ctx, const dfx_frame_desc* desc, uint32_t feature_flags);
DFX_API dfx_status dfx_postfx_execute(dfx_postfx* ctx, const dfx_postfx_render_attribs* attribs);
DFX_API dfx_status dfx_postfx_get_plane(const dfx_postfx* ctx, int32_t id, dfx_plane* out);
DFX_API dfx_status dfx_postfx_get_frame_desc(const dfx_postfx* ctx, dfx_frame_desc* out);
DFX_API const dfx_camera_attribs* dfx_postfx_get_camera_attribs_dev(const dfx_postfx* ctx); /* GetCameraAttribsCB */

/* ---- ScreenSpaceAmbientOcclusion (…/ScreenSpaceAmbientOcclusion.hpp:59-136) ---- */
typedef struct dfx_ssao_render_attribs
{
    void*                   stream;
    dfx_postfx*             postfx;  /* pPostFXContext   */
    const dfx_plane*        depth;   /* pDepthBufferSRV  R32F    */
    const dfx_plane*        normal;  /* pNormalBufferSRV RGBA32F (xyz world-space normal) */
    const dfx_ssao_attribs* attribs; /* pSSAOAttribs     */
} dfx_ssao_render_attribs;

DFX_API dfx_status dfx_ssao_create(dfx_ssao** out);
DFX_API void       dfx_ssao_destroy(dfx_ssao* fx);
DFX_API dfx_status dfx_ssao_prepare(dfx_ssao* fx, dfx_postfx* postfx, uint32_t feature_flags);
/* The reference fades the effect in with wall-clock time (AlphaInterpolation, …cpp:793-795). `alpha < 0`
 * restores that behaviour; parity runs pin it (default after create: pinned to 1.0).                            */
DFX_API dfx_status dfx_ssao_set_alpha_interpolation(dfx_ssao* fx, float alpha);
DFX_API dfx_status dfx_ssao_execute(dfx_ssao* fx, const dfx_ssao_render_attribs* attribs);
DFX_API dfx_status dfx_ssao_get_plane(const dfx_ssao* fx, int32_t id, dfx_plane* out);

/* ---- ScreenSpaceReflection (…/ScreenSpaceReflection.hpp:64-139) ---- */
typedef struct dfx_ssr_render_attribs
{
    void*                  stream;
    dfx_postfx*            postfx;
    const dfx_plane*       color;     /* pColorBufferSRV    RGBA32F */
    const dfx_plane*       depth;     /* pDepthBufferSRV    R32F    */
    const dfx_plane*       normal;    /* pNormalBufferSRV   RGBA32F */
    const dfx_plane*       material;  /* pMaterialBufferSRV RGBA32F */
    const dfx_plane*       motion;    /* pMotionVectorsSRV  RG32F   */
    const dfx_ssr_attribs* attribs;   /* pSSRAttribs        */
} dfx_ssr_render_attribs;

DFX_API dfx_status dfx_ssr_create(dfx_ssr** out);
DFX_API void       dfx_ssr_destroy(dfx_ssr* fx);
DFX_API dfx_status dfx_ssr_prepare(dfx_ssr* fx, dfx_postfx* postfx, uint32_t feature_flags);
DFX_API dfx_status dfx_ssr_set_alpha_interpolation(dfx_ssr* fx, float alpha);
DFX_API dfx_status dfx_ssr_execute(dfx_ssr* fx, const dfx_ssr_render_attribs* attribs);
DFX_API dfx_status dfx_ssr_get_plane(const dfx_ssr* fx, int32_t id, dfx_plane* out);

/* ---- Bloom (…/Bloom.hpp:60-114) ---- */
typedef struct dfx_bloom_render_attribs
{
    void*                    stream;
    dfx_postfx*              postfx;
    const dfx_plane*         color;   /* pColorBufferSRV RGBA32F */
    const dfx_bloom_attribs* attribs; /* pBloomAttribs   */
} dfx_bloom_render_attribs;

DFX_API dfx_status dfx_bloom_create(dfx_bloom** out);
DFX_API void       dfx_bloom_destroy(dfx_bloom* fx);
DFX_API dfx_status dfx_bloom_prepare(dfx_bloom* fx, dfx_postfx* postfx, uint32_t feature_flags);
DFX_API dfx_status dfx_bloom_set_alpha_interpolation(dfx_bloom* fx, float alpha);
DFX_API dfx_status dfx_bloom_execute(dfx_bloom* fx, const dfx_bloom_render_attribs* attribs);
DFX_API dfx_status dfx_bloom_get_plane(const dfx_bloom* fx, int32_t id, dfx_plane* out);
/* Bloom + final ToneMap(+sRGB) with the last two kernels fused; writes `ldr_out`, does not update the bloom output plane. */
DFX_API dfx_status dfx_bloom_execute_tonemapped(dfx_bloom* fx, const dfx_bloom_render_attribs* attribs, const dfx_tonemap_attribs* tonemap,
                                                float ave_log_lum, int32_t convert_to_srgb, const dfx_plane* ldr_out);

/* ---- DepthOfField (PostProcess/DepthOfField/interface/DepthOfField.hpp:59-125) ---- */
typedef struct dfx_dof dfx_dof;
typedef struct dfx_dof_render_attribs
{
    void*                  stream;
    dfx_postfx*            postfx;  /* camera (lens fields included), frame index, closest motion */
    const dfx_plane*       color;   /* pColorBufferSRV RGBA32F */
    const dfx_plane*       depth;   /* pDepthBufferSRV R32F    */
    const dfx_dof_attribs* attribs; /* pDOFAttribs             */
} dfx_dof_render_attribs;
typedef enum dfx_dof_plane_id
{
    DFX_DOF_PLANE_OUTPUT        = 0,  /* == GetDepthOfFieldTextureSRV(): combined colour, alpha of the input kept */
    DFX_DOF_PLANE_COC           = 1,  /* D1                                                   */
    DFX_DOF_PLANE_COC_TEMPORAL  = 2,  /* D2, current frame's slot (temporal smoothing only)   */
    DFX_DOF_PLANE_DILATION_MIP0 = 10, /* +k : dilation level k (0..3); level 3 is blurred     */
    DFX_DOF_PLANE_PREFILTERED0  = 20, /* +i : foreground (0) / background (1) after D9        */
    DFX_DOF_PLANE_BOKEH0        = 22  /* +i : foreground (0) / background (1) after D10       */
} dfx_dof_plane_id;
DFX_API dfx_status dfx_dof_create(dfx_dof** out);
DFX_API void       dfx_dof_destroy(dfx_dof* fx);
DFX_API dfx_status dfx_dof_prepare(dfx_dof* fx, dfx_postfx* postfx, uint32_t feature_flags);
DFX_API dfx_status dfx_dof_set_alpha_interpolation(dfx_dof* fx, float alpha);
DFX_API dfx_status dfx_dof_execute(dfx_dof* fx, const dfx_dof_render_attribs* attribs);
DFX_API dfx_status dfx_dof_get_plane(const dfx_dof* fx, int32_t id, dfx_plane* out);

/* ---- TemporalAntiAliasing (…/TemporalAntiAliasing.hpp:62-156) ---- */
typedef struct dfx_taa_render_attribs
{
    void*                  stream;
    dfx_postfx*            postfx;
    const dfx_plane*       color;   /* pColorBufferSRV RGBA32F */
    const dfx_taa_attribs* attribs; /* pTAAAttribs     */
    uint32_t               accumulation_buffer_idx;
} dfx_taa_render_attribs;

DFX_API dfx_status dfx_taa_create(dfx_taa** out);
DFX_API void       dfx_taa_destroy(dfx_taa* fx);
DFX_API dfx_status dfx_taa_prepare(dfx_taa* fx, dfx_postfx* postfx, uint32_t feature_flags, uint32_t accumulation_buffer_idx);
DFX_API dfx_status dfx_taa_execute(dfx_taa* fx, const dfx_taa_render_attribs* attribs);
/* TAA with the compose step evaluated on the fly (attribs->color = un-composed scene colour; ssr / ao may be NULL). */
DFX_API dfx_status dfx_taa_execute_composed(dfx_taa* fx, const dfx_taa_render_attribs* attribs, const dfx_plane* ssr, const dfx_plane* ao,
                                            float ssr_scale, float ssao_scale);
DFX_API dfx_status dfx_taa_get_plane(const dfx_taa* fx, int32_t id, uint32_t accumulation_buffer_idx, dfx_plane* out);
DFX_API dfx_status dfx_taa_get_jitter_offset(const dfx_taa* fx, uint32_t accumulation_buffer_idx, float out_jitter[2]);

/* ---- CoordinateGridRenderer (Components/interface/CoordinateGridRenderer.hpp:55-189) ---- */
typedef struct dfx_coordinate_grid dfx_coordinate_grid;
typedef struct dfx_coordinate_grid_render_attribs
{
    void*                              stream;         /* stands in for pDeviceContext                                   */
    const dfx_plane*                   color;          /* pColorRTV, RGBA32F, blended in place                           */
    const dfx_plane*                   depth;          /* pDepthSRV, R32F                                                */
    const dfx_camera_attribs*          camera;         /* pCamera: host pointer, uploaded to the effect's own buffer     */
    const dfx_camera_attribs*          camera_dev;     /* pCameraAttribsCB: device pointer; used instead when not NULL   */
    uint32_t                           feature_flags;  /* DFX_GRID_FEATURE_FLAG_*                                        */
    const dfx_coordinate_grid_attribs* attribs;        /* pAttribs (host pointer)                                        */
} dfx_coordinate_grid_render_attribs;
DFX_API dfx_status dfx_coordinate_grid_create(dfx_coordinate_grid** out);
DFX_API void       dfx_coordinate_grid_destroy(dfx_coordinate_grid* fx);
/* CoordinateGridRenderer::Render (CoordinateGridRenderer.cpp:60-103): G1 on the whole frame. */
DFX_API dfx_status dfx_coordinate_grid_render(dfx_coordinate_grid* fx, const dfx_coordinate_grid_render_attribs* attribs);

/* ---- DepthRangeCalculator (Components/interface/DepthRangeCalculator.hpp:62-176) ---- */
typedef struct dfx_depth_range dfx_depth_range;
/* read_back != 0 = CreateInfo::ReadBackData: every compute also copies the range to a pinned host slot (four to start with; one more
 * whenever every slot still has a copy in flight, as the reference's read-back queue adds a staging buffer). The device buffer starts
 * as all zeros. */
DFX_API dfx_status dfx_depth_range_create(int32_t read_back, dfx_depth_range** out);
DFX_API void       dfx_depth_range_destroy(dfx_depth_range* fx);
/* ComputeRange: dfx_pass_depth_range on `depth` with cameras_dev[0] into the effect's buffer, then (with read_back) the copy to a free
 * host slot. */
DFX_API dfx_status dfx_depth_range_compute(dfx_depth_range* fx, void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* depth);
/* GetDepthRangeBuffer: the device buffer (4 floats, dfx_scene_depth_range), valid until destroy. */
DFX_API float* dfx_depth_range_get_buffer(const dfx_depth_range* fx);
/* GetDepthRange: the range of the latest compute whose copy has completed (all zeros before the first one; a copy that completes
 * after a newer one does not replace it). poll != 0 first checks the
 * copies in flight (cudaEventQuery; it never waits); poll == 0 returns what the last poll found. */
DFX_API dfx_status dfx_depth_range_get_range(dfx_depth_range* fx, int32_t poll, dfx_scene_depth_range* out);

/* ============================================================================================================ */
/* Ingest / egress in the reference's render-target formats (Hydrogent/src/Tasks/HnBeginFrameTask.cpp:63-69: scene colour
 * and normal RGBA16_FLOAT, motion RG16_FLOAT, material RG8_UNORM; the final target is an 8-bit sRGB swap chain). The
 * passes keep fp32 planes in HBM; these two entries convert at the PCIe boundary so that the narrow formats are what
 * travels (30 B/px in, 4 B/px out instead of 64 / 16). Widening is exact.
 *   unpack: RGBA16F -> RGBA32F, RG16F -> RG32F, RG8U -> RGBA32F (x, y = c/255; z = w = 0)
 *   pack  : RGBA32F -> RGBA8U, D3D UNORM rule: saturate, * 255, + 0.5, truncate (NaN -> 0)                        */
DFX_API dfx_status dfx_pass_unpack_plane(void* stream, const dfx_plane* src, const dfx_plane* dst, dfx_rows rows);
DFX_API dfx_status dfx_pass_pack_ldr8(void* stream, const dfx_plane* src_rgba32f, const dfx_plane* dst_rgba8u, dfx_rows rows);

/* ============================================================================================================ */
/* plane helpers (device memory owned by the library; used by the C++ shim and the tests)                       */
DFX_API dfx_status dfx_plane_alloc(int32_t width, int32_t height, int32_t format, dfx_plane* out);
DFX_API void       dfx_plane_free(dfx_plane* p);
DFX_API dfx_status dfx_plane_upload(void* stream, const dfx_plane* dst, const void* host_src, size_t host_pitch_bytes);
DFX_API dfx_status dfx_plane_download(void* stream, const dfx_plane* src, void* host_dst, size_t host_pitch_bytes);
DFX_API dfx_status dfx_plane_fill(void* stream, const dfx_plane* dst, const float value[4]);
DFX_API dfx_status dfx_stream_synchronize(void* stream);

/* Optional per-pass device timing (stands in for the reference's ScopedDebugGroup markers, e.g. ScreenSpaceAmbientOcclusion.cpp:363):
 * while enabled every dfx_pass_* call is bracketed by two CUDA events on its stream. Not thread-safe; one stream at a time. */
DFX_API void       dfx_profile_enable(int32_t on);
DFX_API dfx_status dfx_profile_collect(void);                 /* waits for the recorded events, folds them into per-pass totals */
DFX_API void       dfx_profile_reset(void);
DFX_API int32_t    dfx_profile_count(void);
DFX_API dfx_status dfx_profile_entry(int32_t i, char* name, int32_t name_cap, double* total_ms, int32_t* calls);

/* ============================================================================================================ */
/* 3. chain level: the whole PostProcess chain of one view, one call per frame                                    */
/* ============================================================================================================ */
/* Owns one PostFXContext, SSAO, SSR, TAA, DepthOfField and Bloom object and runs them in the order of the reference's only in-tree
 * integration (Hydrogent/src/Tasks/HnPostProcessTask.cpp: Prepare :591-683, Execute :743-947):
 *   PostFXContext -> SSR -> SSAO -> compose -> TAA -> [DepthOfField] -> Bloom -> ToneMap(+sRGB).
 * The SSAO passes run beside the SSR passes on a second stream, Bloom + ToneMap of frame f beside the front half of frame f+1
 * on a third; in steady state (consecutive frame indices, no history reset, constant attributes) the launches are replayed
 * from CUDA graphs cached per (input planes, ping-pong parity, configuration). Results are bit-identical whichever way a frame
 * is issued. Not thread-safe: one chain per view / stream of frames, like the reference's effect objects. */
#define DFX_CHAIN_STAGE_POSTFX  1u
#define DFX_CHAIN_STAGE_SSR     2u
#define DFX_CHAIN_STAGE_SSAO    4u
#define DFX_CHAIN_STAGE_COMPOSE 8u
#define DFX_CHAIN_STAGE_TAA     16u
#define DFX_CHAIN_STAGE_BLOOM   32u
#define DFX_CHAIN_STAGE_TONEMAP 64u
#define DFX_CHAIN_STAGE_ALL     127u

typedef struct dfx_chain_config
{
    dfx_ssao_attribs    ssao;
    dfx_ssr_attribs     ssr;
    dfx_bloom_attribs   bloom;
    dfx_taa_attribs     taa;
    dfx_tonemap_attribs tonemap;
    dfx_dof_attribs     dof;
    uint32_t postfx_flags, ssao_flags, ssr_flags, taa_flags, dof_flags; /* DFX_*_FEATURE_FLAG_* */
    uint32_t stages;      /* DFX_CHAIN_STAGE_* mask                                                                          */
    int32_t  enable_dof;  /* DepthOfField between TAA and Bloom (HnPostProcessTask.cpp:899-909)                                */
    int32_t  fuse;        /* compose inside TAA, ToneMap inside the Bloom composite (same arithmetic, two HBM round trips fewer) */
    int32_t  overlap;     /* async compute on three streams                                                                  */
    int32_t  use_graph;   /* replay steady-state frames from CUDA graphs                                                     */
    int32_t  to_srgb;     /* LinearToSRGB after the tone map (HnCopyFrame.psh:60-62)                                         */
    float    ave_log_lum; /* HnPostProcessTask.hpp:88                                                                        */
    float    ssr_scale, ssao_scale; /* compose: rgb += ssr.rgb * ssr.a * ssr_scale; rgb *= lerp(1, ao, ssao_scale)           */
    int32_t  disable_taa; /* 1: HnPostProcessTask with EnableTAA = false (HnPostProcessTask.cpp:158-187, :652-654, :834-869):
                           * PostFX, SSR, SSAO (+ J), then dfx_pass_compose_final into ldr_out, with the grid over the pixel's own
                           * depth and the selection colours as given. The TAA and BLOOM stage bits, enable_dof and fuse are
                           * ignored; the stages must include COMPOSE and TONEMAP. The first frame with TAA after TAA-off frames
                           * resets TAA's history (its frame index is not consecutive). 0: the chain with TAA.                    */
} dfx_chain_config;

typedef struct dfx_chain_frame
{
    uint32_t                  frame_index;  /* FrameDesc.Index: consecutive, or the histories reset                          */
    int32_t                   defer_post;   /* 1: return without making `stream` wait for Bloom + ToneMap (dfx_chain_join)    */
    const dfx_camera_attribs* curr_camera;  /* host pointers                                                                 */
    const dfx_camera_attribs* prev_camera;
    const dfx_plane*          depth;        /* R32F    */
    const dfx_plane*          prev_depth;   /* R32F    */
    const dfx_plane*          motion;       /* RG32F   */
    const dfx_plane*          normal;       /* RGBA32F */
    const dfx_plane*          color;        /* RGBA32F */
    const dfx_plane*          material;     /* RGBA32F */
    const dfx_plane*          ldr_out;      /* RGBA32F: the tone-mapped frame                                                */
} dfx_chain_frame;

typedef struct dfx_chain_stats
{
    uint64_t frames_eager, frames_replayed, graphs_built, graph_failures;
} dfx_chain_stats;

typedef enum dfx_chain_effect_id
{
    DFX_CHAIN_EFFECT_POSTFX = 0, DFX_CHAIN_EFFECT_SSAO = 1, DFX_CHAIN_EFFECT_SSR = 2, DFX_CHAIN_EFFECT_BLOOM = 3, DFX_CHAIN_EFFECT_TAA = 4, DFX_CHAIN_EFFECT_DOF = 5
} dfx_chain_effect_id;

typedef struct dfx_chain dfx_chain;
DFX_API void       dfx_chain_config_default(dfx_chain_config* config); /* reference struct defaults, Hydrogent's TAA flags, every stage, fused, async, graphs */
DFX_API dfx_status dfx_chain_create(int32_t width, int32_t height, const dfx_chain_config* config /* NULL = defaults */, dfx_chain** out);
DFX_API void       dfx_chain_destroy(dfx_chain* chain);
DFX_API dfx_status dfx_chain_set_config(dfx_chain* chain, const dfx_chain_config* config);
DFX_API dfx_status dfx_chain_get_config(const dfx_chain* chain, dfx_chain_config* out);
/* Runs one frame, ordered after the work already on `stream`; the frame's LDR plane is complete in stream order when the call
 * returns (defer_post = 0) or after dfx_chain_join (defer_post = 1). */
DFX_API dfx_status dfx_chain_execute(dfx_chain* chain, void* stream, const dfx_chain_frame* frame);
DFX_API dfx_status dfx_chain_join(dfx_chain* chain, void* stream);
/* The effect objects (dfx_postfx*, dfx_ssao*, ...) for dfx_*_get_plane / dfx_*_set_alpha_interpolation; owned by the chain. */
DFX_API void*      dfx_chain_effect(dfx_chain* chain, int32_t which /* dfx_chain_effect_id */);
/* The stream Bloom + ToneMap run on when `overlap` is set (to order a read-back after a deferred frame). */
DFX_API void*      dfx_chain_post_stream(dfx_chain* chain);
DFX_API dfx_status dfx_chain_get_stats(const dfx_chain* chain, dfx_chain_stats* out);
/* The coordinate grid and axes in the final copy-frame step (HnPostProcessTask.cpp:397-425, HnCopyFrame.psh:38-58; TAA on).
 * flags != 0: the tone map of every following frame is dfx_pass_copy_frame_grid on the frame's depth and current camera (Bloom
 * then runs its composite unfused and the grid step reads its output); refused when the configured stages lack
 * DFX_CHAIN_STAGE_TONEMAP. flags == 0 (the default): the chain issues exactly the kernels it issues without this call.
 * attribs NULL = the defaults. The settings take effect with the next frame, replayed frames included. With disable_taa the grid is
 * drawn by dfx_pass_compose_final instead (HnPostProcess.psh:246-252: the pixel's own depth, lerp). */
DFX_API dfx_status dfx_chain_set_coordinate_grid(dfx_chain* chain, uint32_t flags, const dfx_coordinate_grid_attribs* attribs);
/* Selection highlighting (HnProcessSelectionTask; HnPostProcess.psh:211-244; HnPostProcessTask.cpp:840-864).
 * attribs != NULL: every following frame runs the compose unfused, J on `selection_depth` (R32F, the chain's size; the plane is
 * read by every frame, so it must stay valid while selection is on) beside SSR, O in place on the composed colour with the outline
 * colours reverse-tone-mapped (dfx_reverse_exp_tone_map with the tone map's fMiddleGray and the chain's ave_log_lum) unless the
 * tone-mapping mode is NONE, then TAA. Refused when the configured stages lack DFX_CHAIN_STAGE_COMPOSE or DFX_CHAIN_STAGE_TAA, or
 * when SelectionOutlineWidth is not positive and finite. With disable_taa, J runs the same way and the outline is drawn by
 * dfx_pass_compose_final with the colours as given; the stages must then include COMPOSE and TONEMAP. A change of selection_id,
 * and switching selection on or off, resets the TAA history on the next frame that runs TAA. attribs NULL (the default): the chain
 * issues exactly the kernels it issues without this call. */
DFX_API dfx_status dfx_chain_set_selection(dfx_chain* chain, const dfx_selection_attribs* attribs, const dfx_plane* selection_depth);
/* The viewer's view mode (HN_VIEW_MODE, DFX_VIEW_MODE_*) from the next frame on, replayed frames included.
 *   SHADED, WHITE_BASE_COLOR (the default): the chain issues exactly the kernels it issues without this call.
 *   Any other mode (a renderer debug view, HnPostProcessTask.cpp:625-654, :788): SSR, SSAO, Bloom and DepthOfField do not run; PostFX
 *   runs only with TAA. For SCENE_DEPTH, EDGE_MAP and MESH_ID the compose is dfx_pass_compose_view; for the others it is the compose
 *   with zero scales. SCENE_DEPTH first runs dfx_pass_depth_range into &cameras_dev[0].fSceneNearZ (HnComputeDepthBoundsTask), so
 *   the compose reads this frame's range. With TAA on, the compose draws the view mode with tone map NONE, no grid and no sRGB, and
 *   the selection with its reverse-tone-mapped colours, into the composed plane; then TAA, then the tone map (with the grid: the grid
 *   step). With disable_taa it writes ldr_out with the tone map, the selection colours as given, the grid and sRGB.
 * A switch does not reset TAA. mesh_id: R32F, the chain's size, read by every MESH_ID frame (it must stay valid while that mode is
 * on); ignored by the other modes. loading_animation_factor: g_Frame.Renderer.LoadingAnimation.Factor, read by SCENE_DEPTH (non-zero
 * skips the rescale). Refuses an unknown mode, MOTION_VECTORS (DFX_ERR_UNSUPPORTED: that view takes the frame's elapsed time, through
 * dfx_chain_set_motion_vector_view), MESH_ID
 * without a chain-sized R32F plane, and a debug view when the stages lack COMPOSE + TAA (or COMPOSE + TONEMAP with disable_taa);
 * dfx_chain_set_config refuses such stages while a debug view is on. */
DFX_API dfx_status dfx_chain_set_view_mode(dfx_chain* chain, int32_t view_mode, const dfx_plane* mesh_id, float loading_animation_factor);
/* The environment-map background (HnRenderEnvMapTask, Hydrogent/src/Tasks/HnRenderEnvMapTask.cpp:120-230): env_map != NULL makes
 * every following frame (replayed frames included) run E (dfx_pass_env_map) as its first kernel, in place on the frame's colour and
 * motion planes, in whichever formats the chain takes them: the sky and its motion are in the G-buffer before PostFX, SSR, SSAO and
 * TAA read it. Motion vectors are always on; the reverse-depth option follows DFX_POSTFX_FEATURE_FLAG_REVERSED_DEPTH; `options`
 * may add DFX_ENV_MAP_OPTION_CONVERT_OUTPUT_TO_SRGB. attribs NULL = HnRenderEnvMapTask's (:162-216): tone map NONE, AverageLogLum
 * 0.3, MipLevel 1, Alpha 0, Scale (1, 1, 1, 1) standing in for the dome light's colour * intensity. E does not run in the
 * SCENE_DEPTH view (HnRenderEnvMapTask::IsActive, :85-94). The map's planes are read by every frame and must stay valid while E is
 * on. env_map NULL switches E off (the default): the chain then issues exactly the kernels it issues without it. Refuses what
 * dfx_pass_env_map refuses about the type, the options, the tone-mapping mode and the map. */
DFX_API dfx_status dfx_chain_set_environment_map(dfx_chain* chain, int32_t type, const dfx_pyramid* env_map, uint32_t options,
                                                 const dfx_env_map_attribs* attribs);
/* The selected prim's bounding box (HnRenderBoundBoxTask, Hydrogent/src/Tasks/HnRenderBoundBoxTask.cpp:107-207): attribs != NULL makes
 * every following frame (replayed frames included) run B (dfx_pass_bound_box) right after E and before PostFX, in place on the
 * frame's colour and motion planes, storing (Color.rgb, 0) as HnRenderBoundBoxTask's PS main does (:75-98). Motion vectors are always
 * on; the reverse-depth option follows DFX_POSTFX_FEATURE_FLAG_REVERSED_DEPTH. B runs in every view mode (the task has no IsActive).
 * attribs NULL switches B off (the default): the chain then issues exactly the kernels it issues without it. Refuses a PatternLength
 * that is not finite and > 0. */
DFX_API dfx_status dfx_chain_set_bound_box(dfx_chain* chain, const dfx_bound_box_attribs* attribs);
/* The motion-vector view (HN_VIEW_MODE_MOTION_VECTORS; HnPostProcessTask.cpp:625-654, :788, :928-943): on != 0 makes every following
 * frame (replayed frames included) run E and B when they are on, J when the selection is on, then F (dfx_pass_compose_final) into
 * ldr_out with zero SSR and SSAO scales, the configured tone map, the selection colours as given, the grid and sRGB, and then the
 * vector field of the frame's motion plane over ldr_out (dfx_pass_vector_field with dfx_vector_field_attribs_hydrogent(width, height,
 * elapsed_time), sRGB = to_srgb), whatever disable_taa says: no PostFX, SSR, SSAO, TAA, Bloom or DepthOfField. elapsed_time is the
 * frame's ElapsedTime in seconds; call again with the next frame's before each frame. The field's two launches are issued after the
 * frame's graph on the caller's stream, so a new elapsed time replays the same graph. The first frame allocates a chain-sized scratch
 * plane. on = 0 leaves the view for SHADED (nothing changes when the view is off); dfx_chain_set_view_mode with any mode leaves it too.
 * The first TAA frame after motion-vector frames resets TAA's history (the frame indices are not consecutive). Refuses a non-finite
 * elapsed_time and, with on != 0, a stage mask without COMPOSE + TONEMAP; dfx_chain_set_config refuses such masks while the view is
 * on. */
DFX_API dfx_status dfx_chain_set_motion_vector_view(dfx_chain* chain, int32_t on, float elapsed_time);

/* ============================================================================================================ */
/* 4. one frame split into row strips over the GPUs of a box (no reference counterpart)                          */
/* ============================================================================================================ */
/* ScreenSpaceReflection S1-S7 (+ the PostFXContext planes they read) on the strip [row_begin[rank], row_begin[rank+1]) of a frame
 * whose other strips are computed by other GPUs (BASELINE.json config 4). Every rank allocates one slab of
 * dfx_ssr_strips_slab_bytes() bytes (dfx_ipc_alloc), maps the other ranks' slabs (dfx_ipc_open) and hands all base addresses
 * over in a dfx_peer_map; all planes live in the slab at offsets that depend on the frame size only. Halo rows of bounded taps are
 * pushed into the neighbours' slabs by a copy kernel and announced through flags in peer memory; the ray march and the temporal
 * pass load what they need beyond the strip from the owning GPU directly (NVLink peer loads); there is no host synchronisation and
 * no NCCL call per frame. The sharded frame is bit-identical to the unsharded one. Several ranks may also live in one process on
 * one device (plain cudaMalloc slabs, one stream per rank): that is how the single-GPU tests cover this path. */
typedef enum dfx_ssr_strips_plane_id
{
    /* inputs: the caller writes its own rows */
    DFX_SSR_STRIPS_PLANE_DEPTH = 0, DFX_SSR_STRIPS_PLANE_PREV_DEPTH_IN = 1, DFX_SSR_STRIPS_PLANE_MOTION = 2, DFX_SSR_STRIPS_PLANE_NORMAL = 3,
    DFX_SSR_STRIPS_PLANE_COLOR = 4, DFX_SSR_STRIPS_PLANE_MATERIAL = 5,
    /* PostFXContext */
    DFX_SSR_STRIPS_PLANE_REPROJECTED_DEPTH = 6, DFX_SSR_STRIPS_PLANE_CLOSEST_MOTION = 7, DFX_SSR_STRIPS_PLANE_PREVIOUS_DEPTH = 8,
    /* SSR */
    DFX_SSR_STRIPS_PLANE_HIZ1 = 9, /* .. HIZ6 = 14 */
    DFX_SSR_STRIPS_PLANE_ROUGHNESS = 15, DFX_SSR_STRIPS_PLANE_MASK = 16, DFX_SSR_STRIPS_PLANE_RADIANCE = 17, DFX_SSR_STRIPS_PLANE_RAYDIR = 18,
    DFX_SSR_STRIPS_PLANE_RESOLVED_RADIANCE = 19, DFX_SSR_STRIPS_PLANE_RESOLVED_VARIANCE = 20, DFX_SSR_STRIPS_PLANE_RESOLVED_DEPTH = 21,
    DFX_SSR_STRIPS_PLANE_RADIANCE_HISTORY0 = 22, DFX_SSR_STRIPS_PLANE_RADIANCE_HISTORY1 = 23, DFX_SSR_STRIPS_PLANE_VARIANCE_HISTORY0 = 24,
    DFX_SSR_STRIPS_PLANE_VARIANCE_HISTORY1 = 25,
    DFX_SSR_STRIPS_PLANE_OUTPUT = 26, /* == GetSSRRadianceSRV(), valid on the own rows */
    DFX_SSR_STRIPS_PLANE_COUNT = 27
} dfx_ssr_strips_plane_id;

typedef struct dfx_ssr_strips dfx_ssr_strips;
DFX_API size_t     dfx_ssr_strips_slab_bytes(int32_t width, int32_t height);
/* peers->base[peers->rank] is this rank's slab (zeroed by this call: make sure no peer touches it before all ranks have returned);
 * blue_noise_tables: the 131,328-byte Sobol + scrambling-tile blob (host memory). */
DFX_API dfx_status dfx_ssr_strips_create(int32_t width, int32_t height, const dfx_peer_map* peers, const uint8_t* blue_noise_tables, dfx_ssr_strips** out);
DFX_API void       dfx_ssr_strips_destroy(dfx_ssr_strips* strips);
DFX_API dfx_status dfx_ssr_strips_plane(const dfx_ssr_strips* strips, int32_t id, dfx_plane* out);
DFX_API dfx_status dfx_ssr_strips_rows(const dfx_ssr_strips* strips, dfx_rows* out);
/* One frame on this rank's strip; every rank of the map calls it for every frame. Ends with an all-rank barrier in stream order. */
DFX_API dfx_status dfx_ssr_strips_execute(dfx_ssr_strips* strips, void* stream, uint32_t frame_index, const dfx_camera_attribs* curr_camera,
                                          const dfx_camera_attribs* prev_camera, const dfx_ssr_attribs* attribs);
/* *timed_out = 1 if a flag wait of an earlier frame gave up after ~2 s (a peer never signalled). Synchronises the device. */
DFX_API dfx_status dfx_ssr_strips_check(const dfx_ssr_strips* strips, int32_t* timed_out);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* DFX_B200_H */
