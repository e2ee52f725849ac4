/*
 * b200pt.h — C-ABI of the wavefront path tracer (libb200pt.so).
 *
 * This is the drop-in boundary for ONE path of nvpro-samples/vk_gltf_renderer: the path tracer
 * backend (reference: src/renderer_pathtracer.{cpp,hpp} + shaders/gltf_pathtrace.slang).  The
 * reference has no FFI: the path sits behind the C++ virtual class `BaseRenderer`
 * (reference src/renderer_base.hpp:33-55).  Every entry point below states which reference
 * interface it stands in for; INTEGRATION.md shows the `B200PathTracer : BaseRenderer` shim a
 * maintainer would add on the reference side.
 *
 * Conventions
 *   - plain C, plain pointers + sizes, no C++/torch types; all structs are POD with the byte
 *     layouts of the reference's host<->device structs (shaders/shaderio.h, gltf_scene_io.h.slang).
 *   - return 0 on success, negative B200PT_E_* on failure (the reference aborts through
 *     NVVK_CHECK; a C ABI cannot, so the code + b200pt_last_error() carry the same information).
 *   - one handle per GPU / per rank; a handle is single-threaded (reference: all BaseRenderer
 *     virtuals run on the render thread, renderer_base.hpp:39-51).
 *   - matrices are glm column-major float[16], exactly as the reference uploads them.
 *   - host pointers are only read during the call (data is copied to HBM); caller keeps ownership.
 */
#ifndef B200PT_H
#define B200PT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PT_ABI_VERSION 5

/* error codes */
#define B200PT_OK 0
#define B200PT_E_INVALID -1     /* bad argument / call order                         */
#define B200PT_E_CUDA -2        /* CUDA runtime error (see b200pt_last_error)        */
#define B200PT_E_NOMEM -3       /* host or device allocation failed                  */
#define B200PT_E_UNSUPPORTED -4 /* feature outside the built path (e.g. physical sky) */
#define B200PT_E_DEVICE -5      /* a kernel raised a device-side error flag (traversal stack overflow): results incomplete */

typedef struct b200pt b200pt_t; /* opaque renderer handle */

/* ---- scene data contract ---------------------------------------------------------------- */

/* reference: shaders/gltf_scene_io.h.slang:41-47 (GltfRenderNode, 136 B) */
typedef struct b200pt_render_node
{
  float   objectToWorld[16];
  float   worldToObject[16];
  int32_t materialID;
  int32_t renderPrimID;
} b200pt_render_node;

/* reference: shaders/gltf_scene_io.h.slang:50-64 (GltfRenderPrimitive + VertexBuffers: the
 * reference stores 7 device addresses; here they are host pointers + the two counts the host
 * side knows from RenderPrimitive::indexCount/vertexCount, src/gltf_scene.cpp:2153-2154).
 * Optional attribute arrays are NULL when the glTF primitive lacks them
 * (src/gltf_scene_vk.cpp:760-851). */
typedef struct b200pt_render_primitive
{
  const uint32_t* indices;      /* 3 per triangle, always widened to u32 */
  const float*    positions;    /* float3 per vertex                     */
  const float*    normals;      /* float3 or NULL                        */
  const uint32_t* colors;       /* packed unorm4x8 or NULL               */
  const float*    tangents;     /* float4 or NULL                        */
  const float*    texCoords[2]; /* float2 or NULL                        */
  uint32_t        triangleCount;
  uint32_t        vertexCount;
} b200pt_render_primitive;

/* reference: shaders/gltf_scene_io.h.slang:121-128 (GltfTextureInfo, 32 B) */
typedef struct b200pt_texture_info
{
  float   uvTransform[6]; /* glm::mat3x2 column-major: c0.xy c1.xy c2.xy */
  int32_t index;          /* glTF texture index, -1 = none               */
  int32_t texCoord;       /* 0 or 1                                      */
} b200pt_texture_info;

/* reference: shaders/gltf_scene_io.h.slang:147-310 (GltfShadeMaterial with every MAT_EXT_*=1,
 * 288 B; anchors 0/32/40/48/52 are static_asserted in src/gltf_material_cache.cpp:46-56). */
typedef struct b200pt_shade_material
{
  float    pbrBaseColorFactor[4];
  float    emissiveFactor[3];
  float    normalTextureScale;
  float    pbrRoughnessFactor;
  float    pbrMetallicFactor;
  int32_t  alphaMode; /* 0 opaque, 1 mask, 2 blend */
  float    alphaCutoff;
  float    occlusionStrength;
  int32_t  doubleSided;
  float    attenuationColor[3];
  float    ior;
  float    transmissionFactor;
  float    thicknessFactor;
  float    attenuationDistance;
  float    clearcoatFactor;
  float    specularColorFactor[3];
  float    clearcoatRoughness;
  float    specularFactor;
  int32_t  unlit;
  float    iridescenceFactor;
  float    iridescenceThicknessMinimum;
  float    iridescenceThicknessMaximum;
  float    iridescenceIor;
  float    anisotropyRotation[2]; /* (sin, cos) */
  float    sheenColorFactor[3];
  float    anisotropyStrength;
  float    sheenRoughnessFactor;
  float    dispersion;
  int32_t  pbrModel; /* 0 metallic-roughness, 1 specular-glossiness */
  float    pbrDiffuseFactor[4];
  float    pbrSpecularFactor[3];
  float    pbrGlossinessFactor;
  float    diffuseTransmissionColor[3];
  float    diffuseTransmissionFactor;
  float    retroreflectionFactor;
  float    multiscatterColorFactor[3];
  float    scatterAnisotropy;
  /* uint16 indices into the texture-info array, 0 = "no texture" */
  uint16_t pbrBaseColorTexture;
  uint16_t normalTexture;
  uint16_t pbrMetallicRoughnessTexture;
  uint16_t emissiveTexture;
  uint16_t occlusionTexture;
  uint16_t transmissionTexture;
  uint16_t thicknessTexture;
  uint16_t clearcoatTexture;
  uint16_t clearcoatRoughnessTexture;
  uint16_t clearcoatNormalTexture;
  uint16_t specularTexture;
  uint16_t specularColorTexture;
  uint16_t iridescenceTexture;
  uint16_t iridescenceThicknessTexture;
  uint16_t anisotropyTexture;
  uint16_t sheenColorTexture;
  uint16_t sheenRoughnessTexture;
  uint16_t pbrDiffuseTexture;
  uint16_t pbrSpecularGlossinessTexture;
  uint16_t diffuseTransmissionTexture;
  uint16_t diffuseTransmissionColorTexture;
  uint16_t retroreflectionTexture;
  uint16_t _pad16[2];
  uint64_t _pad;
} b200pt_shade_material;

/* reference: shaders/gltf_scene_io.h.slang:85-100 (GltfLight, 64 B) */
typedef struct b200pt_light
{
  float   direction[3];
  int32_t type; /* 0 none, 1 directional, 2 spot, 3 point */
  float   position[3];
  float   radius;
  float   color[3];
  float   intensity;
  float   angularSizeOrInvRange;
  float   innerAngle;
  float   outerAngle;
  int32_t _pad;
} b200pt_light;

/* One decoded glTF texture (image + sampler), reference: SceneVk::createTextureImages /
 * getSampler, src/gltf_scene_vk.cpp:909-1098.  Pixels are RGBA8 (4 B/texel), row 0 first.
 * Mip chain is generated on load (reference: GPU blit chain, gltf_scene_vk.cpp:1254-1332). */
typedef struct b200pt_texture
{
  const uint8_t* rgba8;
  int32_t        width;
  int32_t        height;
  int32_t        srgb;      /* 1: decode sRGB->linear on fetch (findSrgbImages, :1102-1154) */
  int32_t        wrapS;     /* glTF enum: 10497 repeat, 33071 clamp, 33648 mirrored         */
  int32_t        wrapT;
  int32_t        magFilter; /* glTF enum 9728 nearest / 9729 linear, -1 default(linear)     */
  int32_t        minFilter; /* glTF enum 9728..9987, -1 default(linear-mip-linear)          */
} b200pt_texture;

/* Everything SceneVk + SceneRtx hand the reference path tracer (Resources::sceneVk.sceneDesc(),
 * sceneRtx.topLevelAS(); reference src/renderer_pathtracer.cpp:667-712,1559). */
typedef struct b200pt_scene_desc
{
  const b200pt_render_node*      renderNodes;
  uint32_t                       numRenderNodes;
  const uint8_t*                 renderNodeVisible; /* NULL = all visible (SceneRtx skips invisible, gltf_scene_rtx.cpp:317-334) */
  const b200pt_render_primitive* renderPrimitives;
  uint32_t                       numRenderPrimitives;
  const b200pt_shade_material*   materials;
  uint32_t                       numMaterials;
  const b200pt_texture_info*     textureInfos; /* element 0 is the reserved "none" slot */
  uint32_t                       numTextureInfos;
  const b200pt_texture*          textures;
  uint32_t                       numTextures;
  const b200pt_light*            lights;
  uint32_t                       numLights;
} b200pt_scene_desc;

/* reference: shaders/shaderio.h:148-168 (SceneFrameInfo, 396 B) */
typedef struct b200pt_frame_info
{
  float   viewMatrix[16];
  float   projInv[16];
  float   viewInv[16];
  float   viewProjMatrix[16];
  float   prevMVP[16];
  float   jitter[2];
  float   imageSize[2];
  int32_t flags; /* B200PT_SCENE_* */
  float   envRotation;
  float   envBlur;
  float   envIntensity;
  float   backgroundColor[3];
  int32_t visualization;
  float   infinitePlaneDistance;
  float   infinitePlaneBaseColor[3];
  float   infinitePlaneMetallic;
  float   infinitePlaneRoughness;
  float   shadowCatcherDarkenAmount;
} b200pt_frame_info;

/* SceneFrameInfoFlags, reference shaders/shaderio.h:138-145 */
#define B200PT_SCENE_IS_ORTHOGRAPHIC (1 << 0)
#define B200PT_SCENE_USE_SOLID_BACKGROUND (1 << 1)
#define B200PT_SCENE_USE_HDR_ENVIRONMENT (1 << 2)
#define B200PT_SCENE_USE_INFINITE_PLANE (1 << 3)
#define B200PT_SCENE_INFINITE_PLANE_SHADOW_CATCHER (1 << 4)

/* PathtracerFlags, reference shaders/shaderio.h:170-175 */
#define B200PT_PT_USE_DLSS (1 << 0)
#define B200PT_PT_USE_OPTIX_DENOISER (1 << 1)
#define B200PT_PT_FIRST_FRAME (1 << 2)

/* reference: shaders/shaderio.h:179-196 (PathtracePushConstant) minus its four device
 * pointers, which the handle owns. 48 B. */
typedef struct b200pt_push_constant
{
  int32_t maxDepth;
  int32_t frameCount;
  float   fireflyClampThreshold;
  float   texGradScale;
  int32_t numSamples;
  int32_t totalSamples;
  float   focalDistance;
  float   aperture;
  int32_t flags;
  float   pixelAngle;
  float   mouseCoord[2];
} b200pt_push_constant;

/* Counters the reference lacks (it reports MSps only, src/benchmarking.cpp:269-279); needed for
 * Mray/s and for the algorithmic-bytes roofline (SURVEY.md §8d). All are totals since the last
 * b200pt_reset_stats(). */
typedef struct b200pt_stats
{
  uint64_t closestRays;   /* Trace() calls (primary + bounce + volume continues)  */
  uint64_t shadowRays;    /* TraceShadow() calls                                   */
  uint64_t shadedHits;    /* surface interactions shaded                           */
  uint64_t pathsStarted;  /* samplePixel() calls                                   */
  uint64_t nodesVisited;  /* BVH nodes fetched (only when built with B200PT_COUNT_TRAVERSAL) */
  uint64_t trisTested;    /* triangles tested  (same)                              */
  double   msTraceClosest; /* CUDA-event time inside k_trace, the closest-hit tree walks (profiling on) */
  double   msTraceShadow;  /* k_shadow, the shadow-ray tree walks                                       */
  double   msShade;        /* k_shade                                                                   */
  double   msOther;       /* raygen + accumulate                                                        */
  double   msTotal;
  uint64_t kernelLaunches;
  uint64_t launchesTraceClosest; /* launches measured into msTraceClosest (profiling on) */
  uint64_t launchesShade;
  uint64_t launchesTraceShadow;
  double   msAnyHit;       /* k_alpha: stochastic alpha / transmission tests on the collected candidates */
  double   msResolve;      /* k_resolve: NEE contribution, Russian roulette, next-bounce queue           */
  uint64_t launchesAnyHit;
  uint64_t launchesResolve;
} b200pt_stats;

/* ---- lifecycle --------------------------------------------------------------------------- */

/* PathTracer::onAttach (reference src/renderer_pathtracer.cpp:80-112): create the device
 * context on `cuda_device`, streams, counters.  No shader compile step exists here: the
 * kernels are AOT-compiled for sm_90a (H100). */
int b200pt_create(b200pt_t** out, int cuda_device);

/* PathTracer::onDetach (reference :163-184). */
void b200pt_destroy(b200pt_t* h);

int         b200pt_abi_version(void);
const char* b200pt_last_error(const b200pt_t* h);

/* Resources::sceneVk / sceneRtx hand-off; stands in for SceneVk::create (gltf_scene_vk.cpp:218-252)
 * + SceneRtx BLAS/TLAS build (gltf_scene_rtx.cpp:140-388) + PathTracer::onSceneInvalidated
 * (renderer_pathtracer.hpp:72).  Copies all arrays to HBM, builds the software wide BVH over the
 * world-space triangles of every visible render node, uploads the textures' mip chains as tiled texels. */
int b200pt_set_scene(b200pt_t* h, const b200pt_scene_desc* scene);

/* ---- opacity micromaps (reference: src/gltf_scene_omm.{hpp,cpp} -- EXT_mesh_opacity_micromap uploaded as VK_EXT_opacity_micromap
 * build input and attached to the BLAS geometry, gltf_scene_rtx.cpp; docs/RENDERING_ARCHITECTURE.md:65-78) ------------------------
 * The arrays are the extension's own: `data` = packed opacity states in the Vulkan micro-triangle order ("bird curve",
 * VK_EXT_opacity_micromap bary2index), `triangles` = VkMicromapTriangleEXT records.  What the RT cores do with them, the software
 * walk does: a micro-triangle whose state is OPAQUE is committed like a FORCE_OPAQUE triangle, a TRANSPARENT one is culled, both
 * WITHOUT the any-hit alpha evaluation and its rand() (raytracer_interface.h.slang:93-100); the two UNKNOWN states still go through
 * the any-hit path.  Nothing is baked here: the host hands over what the asset carries (vk_gltf_renderer_b200/omm.py can bake the
 * arrays from a MASK texture for assets that have none). */
#define B200PT_OMM_FORMAT_2_STATE 1 /* VK_OPACITY_MICROMAP_FORMAT_2_STATE_EXT: 1 bit, 0 transparent / 1 opaque                   */
#define B200PT_OMM_FORMAT_4_STATE 2 /* VK_OPACITY_MICROMAP_FORMAT_4_STATE_EXT: 2 bits, + 2 unknown-transparent / 3 unknown-opaque */
#define B200PT_OMM_INDEX_FULLY_TRANSPARENT (-1) /* VK_OPACITY_MICROMAP_SPECIAL_INDEX_*_EXT */
#define B200PT_OMM_INDEX_FULLY_OPAQUE (-2)
#define B200PT_OMM_INDEX_FULLY_UNKNOWN_TRANSPARENT (-3)
#define B200PT_OMM_INDEX_FULLY_UNKNOWN_OPAQUE (-4)
#define B200PT_OMM_MAX_LEVEL 12

typedef struct b200pt_micromap_triangle /* VkMicromapTriangleEXT */
{
  uint32_t dataOffset; /* bytes into b200pt_micromap::data */
  uint16_t subdivisionLevel;
  uint16_t format;
} b200pt_micromap_triangle;

typedef struct b200pt_micromap /* one entry of the extension's root micromaps[] (gltf_scene_omm.cpp:180-250) */
{
  const uint8_t*                  data;
  uint64_t                        dataSize;
  const b200pt_micromap_triangle* triangles;
  uint32_t                        numTriangles;
} b200pt_micromap;

typedef struct b200pt_primitive_omm /* SceneOmm::PrimitiveOmm (gltf_scene_omm.hpp:52-60): keyed by renderPrimID */
{
  uint32_t       renderPrimID;
  uint32_t       micromap;     /* index into micromaps[]                                                          */
  uint32_t       baseTriangle; /* micromapBaseTriangle, added to every non-negative index                         */
  const int32_t* indices;      /* one per triangle of the primitive (or a special index < 0); NULL = identity     */
  uint32_t       numIndices;   /* length of `indices` (>= the primitive's triangleCount), 0 with NULL             */
} b200pt_primitive_omm;

/* SceneOmm::create.  Copies the arrays; they take effect at the next b200pt_set_scene (like SceneRtx consuming them at BLAS build).
 * num_prims == 0 removes them.  B200PT_E_INVALID on out-of-range indices / offsets, formats other than the two above or levels
 * beyond B200PT_OMM_MAX_LEVEL (checked again against the primitives' triangle counts in b200pt_set_scene). */
int b200pt_set_opacity_micromaps(b200pt_t* h, const b200pt_micromap* micromaps, uint32_t num_micromaps, const b200pt_primitive_omm* prims, uint32_t num_prims);

/* Which builder b200pt_set_scene uses for the three trees (closest-hit, opaque-only, non-opaque): 0 = the host builder (binned
 * SAH + optimal 8-wide collapse + axis maps, csrc/bvh.cpp; default, the better tree), 1 = the DEVICE builder (LBVH: Morton sort,
 * Karras hierarchy, bottom-up fit, level-wise collapse, csrc/lbvh.cuh; built in milliseconds, ~20-30 % more node visits).
 * Either tree can be refitted by b200pt_update_transforms.  Takes effect at the next b200pt_set_scene.  Reference: SceneRtx's
 * driver-side BLAS / TLAS builds, src/gltf_scene_rtx.cpp:173-388.  b200pt_bvh_build_ms: wall time of the last scene's builds. */
int b200pt_set_bvh_builder(b200pt_t* h, int kind);
int b200pt_bvh_build_ms(b200pt_t* h, double* ms);

/* Animation feed, rigid part: the render nodes' transforms changed (same nodes, same primitives and materials; the reference
 * updates its TLAS instance matrices and refits: SceneRtx::updateTopLevelAS, src/gltf_scene_rtx.cpp:416-503).  nodes must hold
 * the scene's numRenderNodes entries with the new objectToWorld / worldToObject.  Every triangle record is recomputed on the
 * device and the wide BVHs are refitted bottom-up (topology kept); a refitted tree answers every ray exactly like a freshly
 * built one.  Synchronous. */
int b200pt_update_transforms(b200pt_t* h, const b200pt_render_node* nodes, uint32_t num_nodes);

/* Animation feed, rigid part ON THE DEVICE: the node hierarchy's world matrices are propagated level by level and the render nodes
 * (objectToWorld, worldToObject = inverse, materialID, renderPrimID) rewritten from them, then the trees are refitted -- the host
 * uploads only the nodes' LOCAL matrices per frame.  Reference: shaders/world_matrix_propagate.comp.slang:27-42 (one dispatch per
 * topological BFS level), shaders/update_render_instances.comp.slang:42-66, structs shaders/world_matrix_io.h.slang:29-69
 * (PropagateWorldMatricesPushConstant, RenderNodeGpuMapping, UpdateRenderInstancesPushConstant).
 * b200pt_set_node_hierarchy (after b200pt_set_scene; copied): parentIndices[numNodes] (-1 = root), topoNodeOrder[numNodes] in BFS
 * order with levelOffsets[numLevels + 1] delimiting the levels, one mapping per render node of the scene (in render-node order) and
 * optional per-render-node instance matrices (glm mat4 bytes; NULL = identity).
 * b200pt_update_node_matrices: localMatrices[numNodes x 16] (glm mat4 bytes).  Synchronous.  Arithmetic order: csrc/animate.cuh. */
typedef struct b200pt_render_node_mapping /* RenderNodeGpuMapping */
{
  int32_t nodeID;
  int32_t pad0;
  int32_t materialID;
  int32_t renderPrimID;
} b200pt_render_node_mapping;

typedef struct b200pt_node_hierarchy
{
  uint32_t                          numNodes;
  uint32_t                          numLevels;
  const int32_t*                    parentIndices;
  const int32_t*                    topoNodeOrder;
  const uint32_t*                   levelOffsets;
  const b200pt_render_node_mapping* mappings;          /* numRenderNodes of the current scene */
  const float*                      instLocalMatrices; /* numRenderNodes x 16 or NULL */
} b200pt_node_hierarchy;

int b200pt_set_node_hierarchy(b200pt_t* h, const b200pt_node_hierarchy* hierarchy);
int b200pt_update_node_matrices(b200pt_t* h, const float* local_matrices);

/* Scene edits without a rebuild of the scene (GltfRenderer::updateSceneChanges, src/renderer.cpp:2269-2362).  After any sequence
 * of edits the handle renders exactly what a fresh handle renders when b200pt_set_scene gets the edited description (same BVH
 * builder, same animation / hierarchy / micromap calls).  Each call first launches a pending frame batch and waits for the frames
 * in flight; every check runs before the first device write, so a refused call (or B200PT_E_NOMEM) leaves the scene as it was.
 * Accumulation is not reset (restart it with frameCount, as after a transform update).  The trees are rewritten in place when the
 * visible set stays and no visible triangle changes between opaque and any-hit; otherwise they are rebuilt with the handle's
 * builder from the primitives' current vertices and the nodes' current transforms (an animated pose stays).  Synchronous.
 *
 * b200pt_update_materials: both tables, as MaterialCache::buildFromMaterials produces them (num_materials must be the scene's;
 *   the texture-info count may change, the texture images may not).  Checked like b200pt_set_scene's materials.
 * b200pt_update_node_materials: every render node's materialID (-1 = material 0), the KHR_materials_variants switch
 *   (Scene::setCurrentVariant); also rewrites the node hierarchy's mappings, which b200pt_update_node_matrices applies.
 * b200pt_update_lights: the light array; the count may change.
 * b200pt_set_node_visibility: one flag per render node, as b200pt_scene_desc::renderNodeVisible. */
int b200pt_update_materials(b200pt_t* h, const b200pt_shade_material* materials, uint32_t num_materials, const b200pt_texture_info* texture_infos,
                            uint32_t num_texture_infos);
int b200pt_update_node_materials(b200pt_t* h, const int32_t* material_ids, uint32_t num_nodes);
int b200pt_update_lights(b200pt_t* h, const b200pt_light* lights, uint32_t num_lights);
int b200pt_set_node_visibility(b200pt_t* h, const uint8_t* visible, uint32_t num_nodes);

/* Animation feed, deforming part: morph-target blending and skeletal skinning of render primitives' vertex arrays ON THE DEVICE
 * (shaders/morph.comp.slang:29-70, shaders/skinning.comp.slang:27-70, push constants shaders/animation_io.h.slang:29-59), as
 * SceneAnimationVk::createAnimationResources / cmdUpdateAnimation drive them (src/gltf_scene_animation_vk.cpp:120-260, 396-592).
 *
 * b200pt_set_animation uploads the static inputs once (base arrays, deltas, weights / joints; all copied) for the primitives of
 * the CURRENT scene (call it after b200pt_set_scene; the next b200pt_set_scene drops them).  vertexCount must equal the
 * primitive's.  Normals / tangents are processed only when the task AND the primitive carry them (shader: hasNormals /
 * hasTangents, host: vb.normal.buffer / vb.tangent.buffer).
 *
 * b200pt_animate is one cmdUpdateAnimation: the per-frame inputs are the concatenations, in task order, of every morph
 * task's target weights (mesh.weights, :445-458), every skin task's joint matrices (glm mat4 bytes, 16 floats per joint:
 * inverse(meshNode) * jointNode * inverseBind, :470-483) and normal matrices (glm mat3 bytes, 9 floats per joint:
 * transpose(inverse(mat3(joint)))).  All morph kernels run, then all skin kernels (a primitive that is both morphed and skinned
 * is skinned from its morphed arrays, :545-556), the per-triangle shade records of the touched primitives are re-gathered, and
 * the trees are refitted like b200pt_update_transforms does (the BLAS update the reference records next).  Synchronous.
 * Arithmetic order is pinned in csrc/animate.cuh and restated in oracle/animation.py. */
typedef struct b200pt_morph_task /* MorphPushConstant minus the per-frame / output pointers */
{
  uint32_t     renderPrimID;
  uint32_t     vertexCount;
  uint32_t     numTargets;
  uint32_t     _pad;
  const float* basePositions;  /* vertexCount x 3                                  */
  const float* baseNormals;    /* vertexCount x 3 or NULL                          */
  const float* baseTangents;   /* vertexCount x 4 or NULL                          */
  const float* positionDeltas; /* numTargets x vertexCount x 3                     */
  const float* normalDeltas;   /* numTargets x vertexCount x 3 or NULL             */
  const float* tangentDeltas;  /* numTargets x vertexCount x 3 or NULL             */
} b200pt_morph_task;

typedef struct b200pt_skin_task /* SkinPushConstant minus the per-frame / output pointers */
{
  uint32_t       renderPrimID;
  uint32_t       vertexCount;
  uint32_t       numJoints;
  uint32_t       _pad;
  const float*   basePositions; /* vertexCount x 3                                 */
  const float*   baseNormals;   /* vertexCount x 3 or NULL                         */
  const float*   baseTangents;  /* vertexCount x 4 or NULL                         */
  const float*   weights;       /* vertexCount x 4 (WEIGHTS_0)                     */
  const int32_t* joints;        /* vertexCount x 4 (JOINTS_0 widened to int32)     */
} b200pt_skin_task;

int b200pt_set_animation(b200pt_t* h, const b200pt_morph_task* morphs, uint32_t num_morphs, const b200pt_skin_task* skins, uint32_t num_skins);
int b200pt_animate(b200pt_t* h, const float* morph_weights, const float* joint_matrices, const float* normal_matrices);

/* nvvk::HdrIbl::loadEnvironment (external; reference call site src/renderer.cpp:1994-1996):
 * takes the decoded lat-long image (RGB float, row 0 = +Y pole), builds the alias table
 * (EnvAccel) and stores the per-texel pdf in alpha.  Returns the integral the reference exposes
 * as HdrIbl::getIntegral() through *integral_out (may be NULL). */
int b200pt_set_environment(b200pt_t* h, const float* rgb, int width, int height, float* integral_out);

/* BaseRenderer::onResize (reference src/renderer_base.hpp:43): (re)allocates the RGBA32F
 * accumulation image (Resources::eImgRendered) and the path-state pool.
 * tile_y0/tile_rows select the rows this handle renders (multi-GPU framebuffer tiling; the
 * reference is single-GPU: pass 0,height).  Seeds always use global pixel coordinates. */
int b200pt_resize(b200pt_t* h, int width, int height, int tile_y0, int tile_rows);

/* Same as b200pt_resize, but the handle's tile is every `world`-th band of `band_rows` rows: global row
 * y belongs to rank (y / band_rows) % world, local row l maps to y = ((l / band_rows) * world + rank) * band_rows
 * + l % band_rows.  Interleaving balances expensive and cheap image regions across GPUs (SURVEY.md section 8e).
 * height must be a multiple of band_rows * world.  Seeds still use global pixel coordinates. */
int b200pt_resize_interleaved(b200pt_t* h, int width, int height, int band_rows, int world, int rank);

/* BaseRenderer::onRender (reference src/renderer_pathtracer.cpp:500-614): one frame =
 * pc->numSamples paths per pixel accumulated into the RGBA32F image exactly like
 * processPixel (shaders/gltf_pathtrace.slang:546-630).  Asynchronous on the handle's stream. */
int b200pt_render_frame(b200pt_t* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc);

/* Blocks until all submitted frames are done (vkQueueWaitIdle analogue). */
int b200pt_synchronize(b200pt_t* h);

/* gBuffers[eImgRendered] access: device pointer to the tile's RGBA32F rows (tile_rows x width),
 * or a copy of it into host memory. */
int b200pt_get_accum_device(b200pt_t* h, float** dev_rgba32f, size_t* num_floats);
int b200pt_read_accum(b200pt_t* h, float* host_rgba32f, size_t num_floats);

/* gBuffers[eImgSelection] + the depth image, written on the first frame of an accumulation only (the frame whose push
 * constants carry B200PT_PT_FIRST_FRAME; reference shaders/gltf_pathtrace.slang:604-616): per pixel of the tile the object
 * id of the selection ray (pixel centre, IRaytracer::TraceLow: all geometry opaque, no culling; render node index + 1,
 * 0 = miss; traceSelectionRay, shaders/pathtrace_functions.h.slang:813-820) and the NDC depth (Vulkan [0,1], 1 = far / miss)
 * of the last sample's first hit.  Either pointer may be NULL. */
int b200pt_read_selection(b200pt_t* h, uint32_t* host_object_ids, float* host_ndc_depth, size_t num_pixels);
int b200pt_get_selection_device(b200pt_t* h, uint32_t** dev_object_ids, float** dev_ndc_depth);

/* Denoiser guide image (OutputImage::eOptixAlbedoNormal, shaders/gltf_pathtrace.slang:240-263, 653-670; the buffer
 * OptiXDenoiser::eGBufferAlbedoNormal of src/renderer_pathtracer.cpp:698): per pixel float4(guide albedo.rgb, asfloat(normal)) of
 * the newest sample's first hit -- base colour as the reference's float16_t guide fields hold it, the shading normal taken to
 * camera space by mul(float3x3(viewMatrix), N), normalised and compressed to 32 bits (nvshaders' compressUnitVec: octahedral,
 * 2 x 16 bits; restated, external); (0, 0, 1) where the primary ray missed.  Written by every frame whose push constants carry
 * B200PT_PT_USE_OPTIX_DENOISER, which requires b200pt_set_guide_outputs(h, 1) (the path pools grow by 32 bytes per slot; calling it
 * re-allocates them like b200pt_resize). */
int b200pt_set_guide_outputs(b200pt_t* h, int enable);
int b200pt_read_guide(b200pt_t* h, float* host_albedo_normal, size_t num_floats);
int b200pt_get_guide_device(b200pt_t* h, float** dev_albedo_normal, size_t* num_floats);

/* The DLSS variant (reference PathtracerFlags::ePtUseDlss, shaders/gltf_pathtrace.slang:564-651): the six guide images the
 * reference's path tracer hands to DLSS Ray Reconstruction (OutputImage::eDlss*, formats of src/dlss.cpp:61-66).  Each plane
 * holds tile_rows x width pixels in its format, so it can be copied into a VkImage of that format:
 *   albedo            RGBA8 UNORM   first-hit base colour (binary16-rounded), alpha 1 where the sample stayed solid
 *   spec_albedo       RGBA16F       EnvBRDFApprox2 of the first hit's dielectric f0 x specular colour, alpha 1
 *   normal_roughness  RGBA16F       world-space shading normal, roughness
 *   motion            RG16F         pixel-space motion vector (camera + instance motion; sky: camera rotation only)
 *   depth             R16F          NDC depth of the first hit (1 = miss)
 *   spec_hit_dist     R16F          distance to the surface behind a glossy reflection of the first hit (65504 = sky, 0 = none)
 * Pixels without a hit read 0 except depth (1) and spec_albedo's alpha (1).  A frame whose push constants carry B200PT_PT_USE_DLSS
 * must have numSamples == 1; its sub-pixel position is 0.5 + frame_info.jitter (no Gaussian jitter is drawn), it REPLACES the
 * accumulation image, never joins a frame batch, and writes the six planes for the newest frame.  It requires
 * b200pt_set_dlss_guides(h, 1), which re-allocates the path pools like b200pt_resize: each slot carries 24 more bytes (previous-
 * frame first-hit position, specular albedo + hit distance as binary16) plus the 32 bytes of the guide records if
 * b200pt_set_guide_outputs is off, and the tile 28 bytes per pixel for the planes.  Instance motion: the first
 * b200pt_update_transforms / b200pt_update_node_matrices after a rendered frame keeps the render nodes' objectToWorld of that
 * frame, and the next frame reprojects its first hits through it; a frame with no update before it sees camera motion only.
 * b200pt_read_dlss_guides copies the planes whose host pointer is not NULL (each *_bytes must hold its plane);
 * b200pt_get_dlss_guides_device returns the device planes and their sizes. */
typedef struct b200pt_dlss_guides
{
  void*  albedo;
  size_t albedo_bytes;
  void*  spec_albedo;
  size_t spec_albedo_bytes;
  void*  normal_roughness;
  size_t normal_roughness_bytes;
  void*  motion;
  size_t motion_bytes;
  void*  depth;
  size_t depth_bytes;
  void*  spec_hit_dist;
  size_t spec_hit_dist_bytes;
} b200pt_dlss_guides;
int b200pt_set_dlss_guides(b200pt_t* h, int enable);
int b200pt_read_dlss_guides(b200pt_t* h, const b200pt_dlss_guides* out);
int b200pt_get_dlss_guides_device(b200pt_t* h, b200pt_dlss_guides* out);

/* Tone mapping + 8-bit encode of the accumulation image: what GltfRenderer::tonemap does to gBuffers[eImgRendered] before
 * saveHeadlessOutputImage writes gBuffers[eImgTonemapped] (src/renderer.cpp:992-1054, 557-573).  The compute shader is
 * nvshaders::Tonemapper (nvpro_core2, external to the reference tree): the struct mirrors the controls the reference's UI and
 * Resources::tonemapperData expose, the operators are restated from their publications (csrc/tonemap.cuh) -- parity UNPINNED.
 * method: 0 filmic (Hejl / Burgess-Dawson), 1 Uncharted 2, 2 clip (sRGB), 3 ACES (Hill fit), 4 AgX, 5 Khronos PBR neutral.
 * isActive == 0 stores the clamped linear colour (the reference disables the tonemapper for debug / guide buffers).
 * autoExposure != 0: exposure is multiplied by 0.18 / (log-average luminance of the image), from a 256-bin log2 histogram built
 * on the device (the reference defaults to auto-exposure, src/resources.hpp:212).
 *
 * b200pt_tonemap: this handle's accumulation image (plain row tiles only; an interleaved multi-GPU tile is tonemapped after
 * the gather with b200pt_tonemap_image) -> device RGBA8 (owned by the handle, b200pt_get_tonemapped_device) and, if
 * host_rgba8 != NULL, copied to the host (tile_rows x width x 4 bytes).  exposure_used (may be NULL) receives the final
 * exposure factor.  b200pt_tonemap_image: any device RGBA32F image of width x height -> a device RGBA8 image.  Synchronous. */
typedef struct b200pt_tonemapper
{
  int32_t method;
  int32_t isActive;
  float   exposure;   /* 1 */
  float   brightness; /* 1 */
  float   contrast;   /* 1 */
  float   saturation; /* 1 */
  float   vignette;   /* 0 */
  int32_t autoExposure;
} b200pt_tonemapper;

int b200pt_tonemap(b200pt_t* h, const b200pt_tonemapper* tm, uint8_t* host_rgba8, size_t num_bytes, float* exposure_used);
int b200pt_tonemap_image(b200pt_t* h, const b200pt_tonemapper* tm, const float* dev_rgba32f, int width, int height, uint8_t* dev_rgba8, float* exposure_used);
int b200pt_get_tonemapped_device(b200pt_t* h, uint8_t** dev_rgba8, size_t* num_bytes);

/* Pipelined read-back: enqueue the copy of the image as of the frames submitted so far into (pinned) host memory
 * and return at once; b200pt_wait_read(slot) blocks until that copy has landed.  slot is 0..7; issuing a read on a
 * slot first waits for the slot's previous read.  With frames in flight a caller reads frame f while frame f+1
 * renders (the reference's swapchain / staging-buffer ring plays this role, nvapp frames-in-flight). */
int b200pt_read_accum_async(b200pt_t* h, float* host_rgba32f, size_t num_floats, int slot);
int b200pt_wait_read(b200pt_t* h, int slot);

/* Number of frames whose bounces may overlap on the device (1..8, default 4; 1 = strictly serial frames).
 * Each lane owns a path pool (176 B per pixel of the tile), so the pool is rebuilt: call before b200pt_resize
 * or expect the accumulation image to be cleared like a resize does. */
int b200pt_set_frames_in_flight(b200pt_t* h, int n);

/* Frame batching: up to n (1..64, default 1 = off) consecutive b200pt_render_frame calls whose frame constants are identical and
 * whose push constants only advance the way the host loop advances them (frameCount + 1, totalSamples + numSamples; the
 * first-frame flag on the first only) are collected and run as ONE wavefront of n x pixels paths; the frames are folded into
 * the image in frame order, so the result is bit-identical to unbatched rendering.  A call that does not continue the
 * pending batch flushes it first; b200pt_flush, b200pt_synchronize, the read_* / get_stats / set_* / resize calls flush too.
 * Until then the pending frames are NOT enqueued: a caller that orders its own stream work behind the image (b200pt_stream)
 * must call b200pt_flush first.  Purpose: a multi-GPU tile is 1/N of the frame; batching N frames gives its kernels the size
 * of a single-GPU frame and divides the kernel launches per frame by N (SURVEY.md section 8e "batch several spp per frame on
 * multi-GPU").  Like b200pt_set_frames_in_flight it rebuilds the path pool (n x 264 B per pixel and lane) and clears the image. */
int b200pt_set_frame_batch(b200pt_t* h, int n);
int b200pt_flush(b200pt_t* h);

/* Let the caller own the accumulation storage (e.g. a torch tensor that NCCL all-gathers):
 * dev_rgba32f must hold tile_rows*width*4 floats on the handle's device. NULL restores the
 * internal buffer. */
int b200pt_set_accum_device(b200pt_t* h, float* dev_rgba32f, size_t num_floats);

/* The CUDA stream the handle launches on (cudaStream_t as void*), for event timing by callers. */
void* b200pt_stream(b200pt_t* h);

int b200pt_get_stats(b200pt_t* h, b200pt_stats* out);
int b200pt_reset_stats(b200pt_t* h);
/* enable per-stage CUDA-event timing: event pairs around every launch on the handle's stream,
 * resolved lazily in b200pt_get_stats (no host sync inside a frame) */
int b200pt_set_profiling(b200pt_t* h, int enabled);

/* ---- ray-level entry points (parity tests + traversal micro-benchmarks) ------------------- */

/* Closest-hit traversal of n rays given as 8 floats each (ox,oy,oz,tmin,dx,dy,dz,tmax), all in
 * device memory; writes 6 x 32-bit per ray: t(float), rnodeID, rprimID, primitiveID (int32,
 * -1 on miss), u, v (float) — the reference HitPayload minus the seed
 * (shaders/raytracer_interface.h.slang:36-47).  Semantics of RayQueryRaytracer::Trace
 * (:69-122) incl. back-face culling flags; `seeds` (u32 per ray, device, may be NULL) feeds the
 * stochastic alpha test and is advanced in place. */
int b200pt_trace_closest(b200pt_t* h, const float* dev_rays, uint32_t n, float* dev_hits, uint32_t* dev_seeds);

/* TraceShadow semantics (:139-187): writes rgb transmission (3 floats per ray). */
int b200pt_trace_shadow(b200pt_t* h, const float* dev_rays, uint32_t n, float* dev_transmission, uint32_t* dev_seeds);

/* Hit-state unit-test hook: n rays traced as b200pt_trace_closest traces them, then the shade kernel's hit fetch,
 * getHitState, ray-cone texture gradient and evaluateMaterial in the feature variant frames of the current scene run.
 * in: 16 floats per item (the 8 floats of the ray, isInside, coneWidth, pixelAngle, texGradScale, 4 unused); out: 96 floats
 * per item (see vk_gltf_renderer_b200/shade_io.py); seeds as for b200pt_trace_closest.  Device pointers.
 * B200PT_E_INVALID without a scene or buffers. */
int b200pt_shade_state(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out, uint32_t* dev_seeds);

/* Size in bytes of the traversal structure (nodes, triangles) for the roofline model. */
int b200pt_bvh_info(b200pt_t* h, uint64_t* node_bytes, uint64_t* tri_bytes, uint32_t* num_nodes, uint32_t* num_tris);

/* BSDF unit-test hooks: evaluate/sample n materials on the device.
 * in: per item 48 floats (see vk_gltf_renderer_b200/bsdf_io.py for the packing); device ptrs. */
int b200pt_bsdf_eval(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out);
int b200pt_bsdf_sample(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out);

/* Texture unit-test hook: n lookups against the current scene; device pointers.
 * in: 8 floats per item (see vk_gltf_renderer_b200/tex_io.py); out: 4 floats (rgba) per item.
 * B200PT_E_INVALID without a scene, or if a record's texture-info slot is outside the scene's. */
int b200pt_texture_lookup(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out);

#ifdef __cplusplus
}
#endif
#endif /* B200PT_H */
