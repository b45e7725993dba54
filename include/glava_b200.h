/* glava_b200.h — C ABI of the GPU-native GLava hot path (PCM -> spectrum -> pixels).
 *
 * Drop-in boundary: this is what a GLava maintainer binds instead of
 *   rd_new / rd_update / rd_destroy            (glava/render.h:53-60, glava/render.c:867,1743,2456)
 * for a BATCH of independent PCM streams.  Plain pointers and sizes only; no CUDA or
 * torch types appear in any signature.  All device memory is owned by the handle.
 * See INTEGRATION.md for the glava.c-side stub.
 *
 * Error behaviour: the reference has no error codes; fatal conditions call the
 * overridable fn-ptr `glava_abort` (glava/glava.h:17, glava/glava.c:77-80).  Here every
 * entry point returns 0 on success / negative GLAVA_B200_E* on failure AND reports the
 * message through `glava_b200_set_abort_hook` (default hook: print to stderr, do NOT exit).
 */
#ifndef GLAVA_B200_H
#define GLAVA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GLAVA_B200_OK        0
#define GLAVA_B200_EINVAL   -1   /* bad argument / unsupported configuration */
#define GLAVA_B200_ECONFIG  -2   /* config file / #request error (reference: glava_abort) */
#define GLAVA_B200_ECUDA    -3   /* CUDA runtime failure (no device, OOM, launch error)   */

/* module ids: directory names under shaders/glava/ selected by `#request mod <name>`
 * (render.c:1100-1110) or -m / force_module (glava.c:391) */
enum { GLAVA_B200_MOD_BARS = 0, GLAVA_B200_MOD_RADIAL = 1, GLAVA_B200_MOD_CIRCLE = 2,
       GLAVA_B200_MOD_GRAPH = 3, GLAVA_B200_MOD_WAVE = 4, GLAVA_B200_MOD_TEST = 5 };

/* A colour macro of a module config (e.g. bars.glsl:20, radial.glsl:17, graph.glsl:11):
 *   mode 1  constant (lo)
 *   mode 0  mix(lo, hi, clamp(X / gradient, 0, 1))           — the shipped form, evaluated in closed form
 *   mode 2  any other GLSL expression of the per-pixel variable X (`d`; `pos` in graph) that the config reader could
 *           compile: the module's glava_b200_color_prog at the end of glava_b200_params is evaluated instead. */
typedef struct {
    int   mode;
    float lo[4], hi[4];
    float gradient;
} glava_b200_color;

/* Compiled colour expression: a straight-line program over 8 four-lane float registers (a scalar lives splat in all
 * four lanes, so scalar-vector arithmetic is lane-wise as in GLSL).  The value of the expression is register `result`.
 * Produced by glava_b200_load_config from the macro's text; every instruction is one individually rounded float op. */
enum { GLAVA_B200_COP_SPLAT = 0,   /* dst = imm in every lane                                   */
       GLAVA_B200_COP_VAR,         /* dst = X in every lane                                     */
       GLAVA_B200_COP_LANE,        /* dst.lane[a] = imm                                         */
       GLAVA_B200_COP_SHUF,        /* dst.lane[k] = reg[a].lane[(imm >> 3k) & 7] unless that selector is 7 */
       GLAVA_B200_COP_ADD, GLAVA_B200_COP_SUB, GLAVA_B200_COP_MUL, GLAVA_B200_COP_DIV,   /* dst = a op b */
       GLAVA_B200_COP_MIN, GLAVA_B200_COP_MAX, GLAVA_B200_COP_MOD, GLAVA_B200_COP_STEP,  /* step(edge = a, x = b) */
       GLAVA_B200_COP_NEG, GLAVA_B200_COP_ABS, GLAVA_B200_COP_FLOOR, GLAVA_B200_COP_CEIL, GLAVA_B200_COP_FRACT,
       GLAVA_B200_COP_SQRT, GLAVA_B200_COP_SIN, GLAVA_B200_COP_COS, GLAVA_B200_COP_LOG, GLAVA_B200_COP_SIGN,
       GLAVA_B200_COP_TRUNC,       /* dst = f(a)                                                */
       GLAVA_B200_COP_MIX,         /* dst = a * (1 - c) + b * c,            c = reg[(int) imm]  */
       GLAVA_B200_COP_CLAMP,       /* dst = min(max(a, b), c)                                   */
       GLAVA_B200_COP_SMOOTHSTEP,  /* edges a, b, x = c                                         */
       GLAVA_B200_COP_LT, GLAVA_B200_COP_LE, GLAVA_B200_COP_EQ, GLAVA_B200_COP_NE,   /* dst = (a op b) ? 1 : 0  (> and >= swap operands) */
       GLAVA_B200_COP_AND, GLAVA_B200_COP_OR, GLAVA_B200_COP_NOT,                    /* on 0 / 1 values                                  */
       GLAVA_B200_COP_SELECT,      /* dst = c != 0 ? a : b,                  c = reg[(int) imm]  */
       GLAVA_B200_COP_EXP, GLAVA_B200_COP_EXP2, GLAVA_B200_COP_LOG2,                 /* dst = f(a)               */
       GLAVA_B200_COP_POW,         /* dst = pow(a, b)                                            */
       GLAVA_B200_COP_ATAN2,       /* dst = atan(a, b); atan(x) is compiled as atan(x, 1)        */
       GLAVA_B200_COP_TAN,         /* dst = sin(a) / cos(a)                                      */
       GLAVA_B200_COP_COUNT };
#define GLAVA_B200_COLOR_OPS  64
#define GLAVA_B200_COLOR_REGS 8
typedef struct { uint8_t op, dst, a, b; float imm; } glava_b200_color_op;
typedef struct { int n_ops, result; glava_b200_color_op ops[GLAVA_B200_COLOR_OPS]; } glava_b200_color_prog;

/* Everything rc.glsl / smooth_parameters.glsl / <module>.glsl configure on this path.
 * Field meaning follows the `#request` (render.c:1033-1314) or `#define` named in the
 * comment.  Defaults = the shipped config files. */
typedef struct {
    /* spectrum */
    int   n;                  /* setbufsize (rc.glsl:190): floats per channel, power of two 256..16384 */
    float fft_scale;          /* setfftscale      smooth_parameters.glsl:46 */
    float fft_cutoff;         /* setfftcutoff     :51 */
    float gravity_step;       /* setgravitystep   :67 */
    float ur;                 /* updates / second the gravity step is divided by (render.c:728,2224);
                                 nominal setsamplerate / (setsamplesize / 4) */
    int   avg_frames;         /* setavgframes     :56 (1..16) */
    int   avg_window;         /* setavgwindow     :61 */
    int   accel_fft;          /* setaccelfft      rc.glsl:211 — 0: pipeline A (render.c:2149-2156 float
                                 chain), 1: pipeline B (R16 passes, render.c:2188-2267) */
    int   smooth_pass;        /* setsmoothpass    :78 */
    float smooth_factor;      /* setsmoothfactor  :72 — as the shaders see it: the "%.6f" literal of the injected
                                 `#define _SMOOTH_FACTOR` (render.c:315-324); the config reader rounds accordingly */
    float sample_range;       /* #define SAMPLE_RANGE :42 */
    float sample_scale;       /* #define SAMPLE_SCALE :37 */
    float hybrid_weight;      /* #define SAMPLE_HYBRID_WEIGHT :34 */
    int   sample_mode;        /* #define SAMPLE_MODE: 0 average, 1 maximum, 2 hybrid */
    int   round_formula;      /* #define ROUND_FORMULA: 0 sinusoidal, 1 linear, 2 circular */
    /* raster, common */
    int   module;             /* GLAVA_B200_MOD_* */
    int   w, h;               /* setgeometry w h (rc.glsl:52) */
    int   channels;           /* _CHANNELS: setmirror ? 1 : 2 (render.c:290) */
    int   premultiply_alpha;  /* setopacity "native" (render.c:1036-1040); 0: per-stage GL blending over clear_color */
    /* bars.glsl */
    float bars_width, bars_gap, bars_outline_width, bars_amplify;
    glava_b200_color bars_color;
    int   bars_outline_mode;  /* 0: vec4(COLOR.rgb * 1.5, COLOR.a) (bars.glsl:22), 1: constant, 2: bars_outline_prog */
    float bars_outline[4];
    int   bars_direction, bars_invert, bars_flip, bars_mirror_yx;
    /* radial.glsl */
    float radial_radius, radial_line;
    float radial_line_half;   /* value of the GLSL expression (C_LINE / 2), integer division for an int literal */
    float radial_outline[4];
    int   radial_nbars; float radial_bar_width, radial_amplify;
    glava_b200_color radial_color;
    float radial_rotate; int radial_invert;
    float radial_bar_alias, radial_c_alias, radial_off_x, radial_off_y;
    /* circle.glsl */
    float circle_radius, circle_line, circle_outline[4], circle_amplify, circle_rotate;
    int   circle_invert, circle_fill, circle_smooth;
    /* graph.glsl */
    float graph_vscale; int graph_direction; glava_b200_color graph_color;
    int   graph_draw_outline, graph_draw_highlight; float graph_outline[4]; int graph_invert;
    /* wave.glsl */
    float wave_min_thickness, wave_max_thickness, wave_base_color[4], wave_amplify, wave_outline[4];
    /* request read-backs the caller sizes its audio with (render.h:10-24, glava.c:487-514) */
    int   rate_request;       /* setsamplerate  rc.glsl:203 */
    int   samplesize_request; /* setsamplesize  rc.glsl:181 */
    /* engine knobs (no reference equivalent) */
    int   fb_slots;           /* framebuffers resident per device; 0 = one per stream (default),
                                 K < batch = ring of K (stream s renders into slot s % K) */
    int   lazy_smooth;        /* 1: K5 evaluates only the texels the module samples, and gravity / average state is kept only
                                 for the bins those texels' taps reach (same pixels; glava_b200_textures() / _spectrum() then hold
                                 only those texels / bins, the rest is stale or zero); 0: all n texels.  After a
                                 glava_b200_reconfigure that widens the sampled set (AMPLIFY does not; BAR_WIDTH, geometry,
                                 setsmoothfactor do), the newly reached bins start from the state they had when they were last
                                 updated (zero at creation): their bars fade in over setavgframes updates, like a GLava restart */
    /* optional stages of rd_update that the shipped configuration leaves off */
    int   bufscale;           /* setbufscale (rc.glsl:236, deprecated): box-average `bufscale` PCM samples
                                 before anything else (render.c:1765-1790); textures then have n / bufscale texels */
    int   interpolate;        /* setinterpolate (rc.glsl:131): keyframe lerp between the last two post-transform
                                 buffers (render.c:1792-1809, 2347-2353).  As in the reference it is inactive when
                                 ur / fr > 0.9 (render.c:1761-1763) and for an fft module under setaccelfft
                                 (render.c:2161-2168) */
    float fr;                 /* glava_b200_update calls per second, the reference's measured gl->fr
                                 (render.c:2386); setframerate when > 0; 0 = same as ur */
    int   transform_smooth;   /* `#request transform <uniform> "smooth"` (render.c:1218-1286; transform_smooth, render.c:694-718)
                                 in the module's bind list — the module shaders are not read here, so the position is a parameter:
                                 1 = after "fft" ... "avg": forces the CPU-order chain (pipeline A, render.c:2143-2154);
                                 2 = BEFORE "fft": applied to the (scaled) PCM ring on the CPU side of handle_audio, the fft chain
                                     and setaccelfft's GL passes follow unchanged (render.c:2131-2156) */
    float smooth_distance;    /* setsmooth       (render.c:917,1201) */
    float smooth_ratio;       /* setsmoothratio  (render.c:918,1204) */
    /* compiled colour expressions (mode 2 of the colour they belong to; n_ops == 0 otherwise) */
    glava_b200_color_prog bars_color_prog, bars_outline_prog, radial_color_prog, graph_color_prog;
    /* setbg / setbgf (render.c:1062-1099; rc.glsl:56 `setbg 00000000`): the glClear colour.  Native opacity never shows
     * it (blending is off and every stage writes every pixel); with premultiply_alpha == 0 (setopacity "none" / "xroot")
     * every module stage is blended over it with SRC_ALPHA / ONE_MINUS_SRC_ALPHA (render.c:1467-1470) */
    float clear_color[4];
    /* radial.glsl details appended later (kept at the end so earlier offsets stay put) */
    int   radial_bar_width_int;      /* BAR_WIDTH was written as an integer literal: the shader's `BAR_WIDTH / 2`
                                        (radial/1.frag:62,79,88) is then an integer division */
    float radial_bar_outline_width;  /* BAR_OUTLINE_WIDTH (deprecated, radial.glsl:33-36; default 0) */
    float radial_bar_outline[4];     /* BAR_OUTLINE (default: OUTLINE) */
    int   graph_join_channels;       /* JOIN_CHANNELS (graph.glsl:23): the two halves meet at a common height in the middle */
    int   graph_anti_alias;          /* ANTI_ALIAS (graph.glsl:19): graph/3.frag fades the column steps of the line */
    int   shader_pre_smoothed;       /* what the module's stage-1 shader believes about its audio textures
                                        (`_PRE_SMOOTHED_AUDIO`): 0 = what smooth_pass says (consistent), 1 = "already smoothed"
                                        although the K5 pass is off, 2 = "raw" although K5 ran (smoothed twice).  The reference
                                        gets into 1 / 2 when smooth_parameters.glsl flips setsmoothpass: the module's first
                                        shader header is built before its includes' requests run (render.c:284-293, 312);
                                        the config reader reproduces that */
    int   mirror_input;              /* setmirror as the AUDIO side sees it (r->mirror_input, render.c:1054-1058: the backend mixes
                                        both channels into one, fifo.c:98-102).  `channels` above is what the SHADER sees
                                        (`_CHANNELS`), which bars' `DISABLE_MONO 1` turns back into 2 (bars/1.frag:32-34) while the
                                        rings stay mono.  0 with channels == 1 is treated as 1 (older callers set only channels) */
} glava_b200_params;

/* Stream style: what one stream of a batch overrides of the renderer's look — the `AMPLIFY` (graph: `VSCALE`) and the
 * `@fg` / `@bg` colour binds the shipped module configs route their colours through, i.e. what `--pipe fg / bg` binds
 * give one GLava instance (glava.c:421-436).  `set` is a mask of GLAVA_B200_STYLE_*; a field outside it is ignored.
 *   amplify  bars_amplify / radial_amplify / circle_amplify / graph_vscale / wave_amplify
 *   fg       bars_color, radial_color, graph_color (mode 0 or 1; the module's colour program is dropped);
 *            circle_outline, wave_base_color = fg.lo (mode 1 only).  Mode 1 takes lo, as a constant macro does (hi = lo,
 *            the gradient is kept)
 *   bg       bars: bars_outline_mode = 1, bars_outline = bg; radial: radial_outline and radial_bar_outline;
 *            graph_outline; wave_outline.  circle has no `@bg`
 * The test module has no style.  fg mode 2, a non-finite amplify, bg on circle, fg without bg on bars whose outline is an
 * expression (bars_outline_mode 2) and anything validation refuses are GLAVA_B200_EINVAL. */
#define GLAVA_B200_STYLE_AMPLIFY 1u
#define GLAVA_B200_STYLE_FG      2u
#define GLAVA_B200_STYLE_BG      4u
typedef struct { uint32_t set; float amplify; glava_b200_color fg; float bg[4]; } glava_b200_stream_style;

typedef struct glava_b200 glava_b200;    /* plays the role of struct glava_renderer (render.h:8-30) */

/* Fatal-error hook, the analogue of the `glava_abort` fn-ptr (glava.h:17). NULL restores the default. */
void glava_b200_set_abort_hook(void (*hook)(const char* message));
const char* glava_b200_last_error(void);

/* Shipped-default parameters for a module name ("bars", "radial", "circle", "graph", "wave", "test"). */
int glava_b200_default_params(glava_b200_params* out, const char* module);

/* Config surface — the part of rd_new (render.c:1322-1435) that reads `entry` (rc.glsl) from the
 * first directory in the NULL-terminated `paths` that has it, applies `#request`s, then the
 * NULL-terminated `requests` strings (CLI --request, render.c:1415-1435), then reads
 * smooth_parameters.glsl and <module>.glsl (`#define`s) with user-dir-over-system-dir precedence.
 * `force_module` = the -m option (may be NULL).  paths may be NULL: shipped defaults. */
int glava_b200_load_config(glava_b200_params* out, const char* const* paths, const char* entry,
                           const char* const* requests, const char* force_module);

/* Same, with `--pipe` binds (glava.c:421-436): NULL-terminated "name=value" strings; a config macro written
 * `@name:default` (glsl_ext.c:516-591) takes `value` (#rrggbb[aa] or vec4(...)) when `name` is bound. */
int glava_b200_load_config_binds(glava_b200_params* out, const char* const* paths, const char* entry,
                                 const char* const* requests, const char* force_module, const char* const* binds);

/* Live `--pipe` binds (glava.c:338-411, render.c:1846-2100).  pipe_args: NULL-terminated "NAME[:TYPE]" strings exactly
 * as given to `--pipe` (TYPE one of int, float, bool, vec2, vec3, vec4; default vec4; a NULL-equivalent name is "_"),
 * validated with the reference's messages.  The other arguments are those of glava_b200_load_config and are copied.
 *   _feed    bytes as they arrive on stdin; every complete line `name = value` (or just `value` for the first bind)
 *            is parsed with the reference's rules — prefix match of the name, "#rrggbb[aa]" or "r,g,b,a" for vec4,
 *            true/TRUE/True/1 for bool ... — and its messages ("Bad assignment format", "Variable name not bound",
 *            "Bad format for color string").  Returns the number of binds that took a new value.
 *   _params  the configuration re-evaluated with every `@name:default` macro of a bound name reading the bind's current
 *            value (0 / vec4(0) until its first line, like an unwritten GL uniform).
 *   _apply   _params + glava_b200_reconfigure when a bind changed since the last call: the uniform write of
 *            render.c:2071-2100.  Call once per frame after _feed. */
typedef struct glava_b200_pipe glava_b200_pipe;
glava_b200_pipe* glava_b200_pipe_new(const char* const* paths, const char* entry, const char* const* requests,
                                     const char* force_module, const char* const* pipe_args);
int  glava_b200_pipe_feed(glava_b200_pipe* p, const char* bytes, size_t len);
int  glava_b200_pipe_params(glava_b200_pipe* p, glava_b200_params* out);
int  glava_b200_pipe_bind_count(const glava_b200_pipe* p);
int  glava_b200_pipe_bind(const glava_b200_pipe* p, int index, const char** name, const char** type, float value[4]);
void glava_b200_pipe_free(glava_b200_pipe* p);

/* rd_new (render.h:53-57): build a renderer for `batch` independent streams on CUDA device
 * `device` with the given parameters (from glava_b200_load_config / _default_params). */
glava_b200* glava_b200_new(const glava_b200_params* params, int batch, int device);
/* rd_destroy (render.h:60) */
void glava_b200_destroy(glava_b200* r);

/* Live parameter update — the analogue of a `--pipe` uniform write (render.c:1846-2005): colours, AMPLIFY,
 * gradient, smoothing parameters ... take effect from the next update.  Everything that sizes device state
 * (setbufsize, geometry, module, setaccelfft, setavgframes, fb_slots) must be unchanged.  Invalid parameters leave the
 * renderer as it was.  If building the new tables fails (out of memory), the renderer keeps its previous parameters but
 * has no tables: every update fails until a reconfigure or resize succeeds. */
int  glava_b200_reconfigure(glava_b200* r, const glava_b200_params* params);
int  glava_b200_get_params(const glava_b200* r, glava_b200_params* out);
int  glava_b200_pipe_apply(glava_b200_pipe* p, glava_b200* r);   /* see glava_b200_pipe_new */
int  glava_b200_batch(const glava_b200* r);
const char* glava_b200_module_name(const glava_b200* r);

/* Pinned host memory for the PCM rings handed to glava_b200_update (so the H2D copy is a
 * true async DMA).  Plain malloc'd memory is accepted too, just slower. */
void* glava_b200_host_alloc(size_t bytes);                 /* placed on the NUMA node of the CURRENT CUDA device */
void* glava_b200_host_alloc_on(size_t bytes, int device);  /* ... of `device` (anonymous mapping + mbind + cudaHostRegister;
                                                              plain cudaHostAlloc when the topology is not exposed or
                                                              GLAVA_B200_NO_NUMA is set) */
void  glava_b200_host_free(void* p);
/* NUMA helpers for one-process-per-GPU callers: the node a device hangs off (-1: unknown), and pinning the calling
 * thread to that node's CPUs (what `numactl --cpunodebind` would do; returns the node or -1, nothing changed). */
int   glava_b200_device_numa_node(int device);
int   glava_b200_bind_thread_to_device(int device);

/* rd_update (render.h:58-59; render.c:1743-2417), batched.
 *   lb, rb : HOST, [batch][bsz] float32, ring contents oldest-first, exactly what glava.c:528-537
 *            memcpy's into lb/rb for one stream.  NOT modified (the reference transforms them in
 *            place, render.c:2140-2180).  rb is ignored by `wave` (audio_l only, wave/1.frag:7); for every
 *            other module a NULL rb with modified != 0 is GLAVA_B200_EINVAL.
 *   bsz    : must equal params.n (setbufsize; with setbufscale k the spectrum has n / k entries)
 *   modified: as rd_update's flag; 0 re-rasters the last spectrum (render.c:2268-2272), or, with keyframe
 *            interpolation active, the next interpolated one
 * Copies H2D on a dedicated copy stream (double-buffered staging: the copy of update i+1 overlaps the
 * kernels of update i), runs the fused spectrum kernel and the module raster kernel on the handle's
 * stream.  Returns once the host buffers have been consumed (they may be reused immediately) and the
 * kernels are enqueued; call glava_b200_sync to wait for the frame. */
int glava_b200_update(glava_b200* r, const float* lb, const float* rb, size_t bsz, int modified);
/* Double-buffer contract for callers that must not block: after glava_b200_set_async_input(r, 1) the update calls return
 * once the H2D copy is ENQUEUED; lb / rb must stay untouched until glava_b200_wait_input(r) (or the next glava_b200_sync).
 * A caller alternating between two sets of rings never waits on a copy. */
int glava_b200_set_async_input(glava_b200* r, int enable);
int glava_b200_wait_input(glava_b200* r);
/* same with DEVICE pointers (inputs already resident in HBM).  The kernels read d_lb / d_rb (16-byte aligned) on an INTERNAL
 * non-blocking stream: either the buffers are complete before the call and stay untouched until glava_b200_sync, or the
 * caller orders its own stream with the two event hooks below. */
int glava_b200_update_device(glava_b200* r, const float* d_lb, const float* d_rb, size_t bsz, int modified);
/* ready_event: a cudaEvent_t (as void*) recorded on the producer's stream after d_lb / d_rb were written; the update waits
 * for it on the device.  glava_b200_input_event(): a cudaEvent_t recorded after the kernels that READ the buffers of the
 * updates issued so far — cudaStreamWaitEvent(producer, ev) before overwriting them. */
int   glava_b200_update_device_after(glava_b200* r, const float* d_lb, const float* d_rb, size_t bsz, int modified, void* ready_event);
void* glava_b200_input_event(glava_b200* r);

/* Per-stream `modified` (glava.c:528-537 tests the flag of ITS audio thread; in a batch every stream has its own):
 * modified[s] != 0 = stream s has new audio and runs the whole chain; a stream with 0 keeps its gravity / average state
 * untouched and is re-rastered from its previous texture, exactly what rd_update(modified = false) does for it
 * (render.c:2122, 2268-2272).  All zero / all non-zero are the plain calls above.  After the first uneven update every
 * stream carries its own average-ring cursor; plain modified = 1 calls keep working.  lb / rb rows of unmodified
 * streams are not read by the kernels.  Not available (GLAVA_B200_EINVAL) for an uneven mask while keyframe
 * interpolation is active (setinterpolate with ur / fr <= 0.9: the keyframe rotation belongs to the renderer). */
int glava_b200_update_masked(glava_b200* r, const float* lb, const float* rb, size_t bsz, const uint8_t* modified /* [batch] */);
int glava_b200_update_device_masked(glava_b200* r, const float* d_lb, const float* d_rb, size_t bsz, const uint8_t* modified);
int glava_b200_update_rings_masked(glava_b200* r, const uint8_t* modified);

/* FIFO-compatible ingest (fifo.c:89-110): `frames` new interleaved int16 L,R frames per stream,
 * HOST [batch][frames*2]; slides every stream's device-resident ring and converts s16/65535.f
 * (mono: integer mean first, fifo.c:98-102, when params.mirror_input — or, for callers that only set it, channels == 1).  Then
 * glava_b200_update_rings() runs the update on the resident rings. */
int glava_b200_ingest_fifo(glava_b200* r, const int16_t* chunks, int frames);
/* The PulseAudio backend's ring update (pulse_input.c:146-174): the samples are ALREADY float (PA_SAMPLE_FLOAT32NE, no
 * / 65535), HOST [batch][frames*2] interleaved L,R; params.channels == 1 mixes (l + r) / 2 in float into both rings. */
int glava_b200_ingest_float(glava_b200* r, const float* chunks, int frames);
int glava_b200_update_rings(glava_b200* r, int modified);

int glava_b200_sync(glava_b200* r);

/* Outputs.  Frame layout: RGBA8, [h][w][4] bytes, row 0 = bottom row (GL window coordinates),
 * byte order R,G,B,A. */
int glava_b200_readback(glava_b200* r, int stream, uint8_t* rgba);              /* one stream's frame -> HOST */
int glava_b200_readback_async(glava_b200* r, int stream, uint8_t* rgba);        /* same, asynchronous: the frame is snapshotted on the
                                                                                   handle's stream (D2D) and copied out on a separate
                                                                                   one, under the next update's kernels; rgba (pinned)
                                                                                   is valid after glava_b200_sync */
int glava_b200_readback_fence(glava_b200* r);                                   /* orders later work on glava_b200_cuda_stream() after
                                                                                   the read-backs issued so far (for event timing) */
int glava_b200_spectrum(glava_b200* r, float* out_l, float* out_r);             /* HOST [batch][n]: pipeline-A result
                                                                                   (accel_fft 0) or raw transform_fft output (1);
                                                                                   n / bufscale entries per stream */
int glava_b200_spectrum_size(const glava_b200* r);                              /* entries per channel of spectra / textures */
int glava_b200_textures(glava_b200* r, uint16_t* out_l, uint16_t* out_r);       /* HOST [batch][n] R16 texels the module samples */
const void* glava_b200_framebuffer_device(const glava_b200* r);                 /* DEVICE [fb_slots][h][w] RGBA8 */
void* glava_b200_cuda_stream(const glava_b200* r);                              /* cudaStream_t, for event timing */

/* Offscreen hand-off — the analogues of glava_sizereq / glava_wait / glava_tex (glava.h:22-24, glava.c:244-267) for a
 * consumer (compositor, encoder) that takes frames straight from HBM:
 *   glava_b200_sizereq         thread-safe resize request, applied at the start of the next update (render.c:1811-1830);
 *                              spectrum state is kept, framebuffers and geometry tables are rebuilt.  An invalid
 *                              geometry fails that update and changes nothing; one whose buffers cannot be allocated
 *                              fails it, keeps the old parameters and leaves the renderer refusing updates until a
 *                              reconfigure or resize succeeds
 *   glava_b200_wait_frame      host-blocks until the latest frame is complete (glava_wait)
 *   glava_b200_frame_event     cudaEvent_t recorded after the latest raster: cudaStreamWaitEvent(consumer, ev) orders a
 *                              consumer stream after the frame without a host round trip (glava_tex hands out the GL
 *                              texture id; here the "texture" is glava_b200_frame_device / _framebuffer_device)
 *   glava_b200_framebuffer_ipc cudaIpcMemHandle_t (64 bytes) of the framebuffer array, for a consumer in another
 *                              process (the OBS-plugin situation, glava-obs/entry.c:141-214)
 * The framebuffer is READ-ONLY for consumers, through these pointers and through the IPC mapping alike: the bars, graph
 * and wave rasters skip storing rows that they themselves left at zero in that slot, so a pixel written from outside can
 * survive into later frames.  Copy a frame out before modifying it. */
int   glava_b200_sizereq(glava_b200* r, int w, int h);
int   glava_b200_wait_frame(glava_b200* r);
void* glava_b200_frame_event(const glava_b200* r);
const void* glava_b200_frame_device(const glava_b200* r, int stream);
int   glava_b200_framebuffer_ipc(glava_b200* r, void* handle, size_t handle_bytes);

/* Frame export into the caller's DEVICE buffers (DESIGN.md §4.10), for a consumer that wants frames top-down, opaque or in
 * NV12 (a compositor's surface, an encoder's input) without writing its own flip / composite / convert pass.
 *   glava_b200_export_frames   converts the current frame of streams[i] — exactly what glava_b200_readback(streams[i])
 *                              would return at this point in call order, framebuffer ring included — into dst[i]
 *                              (a device pointer on the renderer's device; streams may repeat).  Every format is
 *                              top-down: output row 0 is framebuffer row h - 1.
 *     GLAVA_B200_EXPORT_RGBA   h rows of w * 4 bytes R,G,B,A, `pitch` bytes apart
 *     GLAVA_B200_EXPORT_BGRA   the same as B,G,R,A (what compositors and NVENC's ARGB input take)
 *     GLAVA_B200_EXPORT_NV12   Y plane of h rows x w bytes, then the interleaved CbCr plane of h / 2 rows x w bytes at
 *                              `uv_offset` (0: pitch * h); BT.709 limited range (or as the colour flags below say) in
 *                              16-bit fixed point (export_core.h),
 *                              chroma from the per-channel average (s + 2) >> 2 of each composited 2x2 block; w and h even
 *     GLAVA_B200_EXPORT_I420   planar 4:2:0 (yuv420p): Y plane of h rows x w bytes at `pitch`, then the Cb and Cr planes of
 *                              h / 2 rows x w / 2 bytes at `pitch / 2`; NV12's arithmetic, so Y equals NV12's Y and Cb / Cr
 *                              the deinterleaved NV12 CbCr plane, bit for bit; w and h even, pitch a multiple of 32
 *     GLAVA_B200_EXPORT_YUV444 planar 4:4:4: Y, Cb and Cr planes of h rows x w bytes at `pitch`; Y as NV12's, Cb / Cr per
 *                              composited pixel with no averaging
 *     GLAVA_B200_EXPORT_P010   10-bit 4:2:0: Y plane of h rows x w little-endian uint16, then the interleaved CbCr plane of
 *                              h / 2 rows x w / 2 (Cb, Cr) uint16 pairs, both at `pitch` (>= 2 w); each sample is the 10-bit
 *                              BT.709 limited-range code (or as the colour flags say) << 6; chroma from the exact per-channel sums of each composited
 *                              2x2 block (export_core.h); w and h even
 *     GLAVA_B200_EXPORT_YUV420P10  planar 10-bit 4:2:0 (ffmpeg's yuv420p10le): Y plane of h rows x w little-endian uint16 at
 *                              `pitch` (>= 2 w), then the Cb and Cr planes of h / 2 rows x w / 2 uint16 at `pitch / 2`;
 *                              each sample is the 10-bit code in its low bits (0..1023): P010's Y and chroma >> 6, bit for
 *                              bit (DESIGN.md §4.16); w and h even, pitch a multiple of 32
 *     GLAVA_B200_EXPORT_YUV444P10  planar 10-bit 4:4:4 (yuv444p10le): Y, Cb and Cr planes of h rows x w uint16 at `pitch`
 *                              (>= 2 w), LSB-aligned; Y as YUV420P10's, Cb / Cr per composited pixel with no averaging
 *     GLAVA_B200_EXPORT_YUV422P    planar 4:2:2 (yuv422p): Y plane of h rows x w bytes at `pitch`, then the Cb and Cr planes
 *                              of h rows x w / 2 bytes at `pitch / 2`; Y as I420's, Cb / Cr of each horizontal pixel pair
 *                              are I420's of the 2x2 block whose two rows are that pair (DESIGN.md §4.18); w even (any h),
 *                              pitch a multiple of 32
 *     GLAVA_B200_EXPORT_YUV422P10  planar 10-bit 4:2:2 (yuv422p10le, what ProRes 422 and DNxHR HQX encoders take): as
 *                              YUV422P with LSB-aligned uint16 samples, Y rows of 2 w bytes and chroma rows of w bytes at
 *                              `pitch / 2`; YUV420P10's arithmetic on the pair, as YUV422P's on I420's
 *     GLAVA_B200_EXPORT_UYVY   packed 4:2:2 (ffmpeg's uyvy422, NDI's UYVY, DeckLink's 2vuy): one plane of h rows x 2 w
 *                              bytes at `pitch`, each pixel pair the bytes Cb, Y0, Cr, Y1 of YUV422P; w even (any h)
 *     GLAVA_B200_EXPORT_YUVA420P   I420 with an alpha plane (ffmpeg's yuva420p, what libvpx-vp9 encodes as WebM with
 *                              transparency): Y, Cb and Cr as I420 places them, then the A plane of h rows x w bytes at
 *                              `pitch`, one Cb to Cr distance past Cr.  Never composited: Y per pixel and the chroma of each
 *                              2x2 block are of the straight (unassociated) colour, the block's colour weighted by alpha,
 *                              and A is the stored alpha (DESIGN.md §4.19); w and h even, pitch a multiple of 32
 *     GLAVA_B200_EXPORT_YUVA444P10 YUV444P10 with an alpha plane (yuva444p10le, what ProRes 4444 encoders take): four
 *                              planes of h rows x w LSB-aligned uint16 at `pitch`, Y, Cb, Cr and A, placed as YUVA420P's;
 *                              YUV444P10's arithmetic on the straight colour, A = (a 1023 + 127) / 255
 *   Under any opacity but native the frame is opaque: the YUVA formats write I420's / YUV444P10's Y, Cb and Cr bytes with
 *   A = 255 (1023).  Zero pixels are transparent black under native opacity.
 *   Where the chroma planes go: NV12 and P010 put the CbCr plane at `uv_offset` from dst[i] (0: pitch * h).  The planar
 *   formats (I420, YUV444, YUV420P10, YUV444P10) put the Cb plane right after the luma, at dst[i] + pitch * h, and
 *   `uv_offset` is the distance from Cb to Cr (0: the Cb plane's own size, so the planes sit back to back as a yuv420p /
 *   yuv444p buffer does); when set it is at least one chroma plane.  YUV422P and YUV422P10 place their planes so too; UYVY
 *   has no chroma plane, and its uv_offset is 0.  The YUVA formats put A one Cb to Cr distance past Cr, so with uv_offset
 *   0 the four planes sit back to back as ffmpeg's yuva420p / yuva444p10le buffers do.  All YUV formats but YUVA420P and
 *   YUVA444P10 are composited (EXPORT_OVER implied); EXPORT_OVER on a YUVA format is GLAVA_B200_EINVAL.
 *   GLAVA_B200_EXPORT_OVER     (implied for the YUV formats) the opaque colour GLava's window shows over `background` (RGB8,
 *                              byte 3 unused): under setopacity "native" (premultiply_alpha) C = min(255, c +
 *                              mul_norm8(bg, 255 - a)) per channel; under any other opacity the stored colour (the window
 *                              ignores alpha and the clear colour already stands in for the desktop).  Alpha becomes 255.
 *                              Without it RGBA / BGRA carry the stored pixels, alpha included (premultiplied under
 *                              native opacity).
 *   GLAVA_B200_EXPORT_STRAIGHT (RGBA / BGRA only, not with EXPORT_OVER) the stored pixel with its colour un-premultiplied,
 *                              what PNG and ffmpeg's rgba / bgra mean: S = a == 0 ? 0 : min(255, (c 255 + a / 2) / a) per
 *                              channel, alpha as stored; re-premultiplying S with the blend path's unorm8 product gives c
 *                              back wherever c <= a (DESIGN.md §4.19).  Under any other opacity than native, EXPORT_OVER's
 *                              bytes.
 *   GLAVA_B200_EXPORT_FULL_RANGE, GLAVA_B200_EXPORT_BT601   the Y'CbCr encoding of every YUV format (DESIGN.md
 *                              §4.15).  Neither: BT.709 limited range.  BT601 takes Kr, Kb = 0.299, 0.114 for BT.709's
 *                              0.2126, 0.0722; FULL_RANGE writes Y = Y', C = 128 + P over 0..255 (10 bits: 1023/255 Y',
 *                              512 + 1023/255 P, clamped to 1023) for limited range's 16 + 219/255 Y', 128 + 224/255 P
 *                              (64 + 876/255 Y', 512 + 896/255 P).  Both: the JFIF encoding JPEG encoders take (nvJPEG's
 *                              YUV input, libjpeg-turbo's raw data, ffmpeg's yuvj420p).  Every grey has Cb = Cr = 128
 *                              (512).  RGBA / BGRA with either bit are GLAVA_B200_EINVAL (no matrix or range).
 *   GLAVA_B200_EXPORT_PQ, GLAVA_B200_EXPORT_HLG   (P010, YUV420P10, YUV444P10 and YUV422P10 only) BT.2020 non-constant-
 *                              luminance Y'CbCr, limited range, with the PQ (SMPTE ST 2084, HDR10) or HLG (ITU-R BT.2100)
 *                              transfer: each R'G'B' colour is shown as SDR graphics at BT.2408's 203 cd/m^2 (BT.1886
 *                              linearisation, BT.709 -> BT.2020 primaries, HLG through the inverse OOTF of a 1000 cd/m^2
 *                              display), so white is Y 573 (PQ) or 721 (HLG) and no channel exceeds 203 cd/m^2: MaxCLL
 *                              <= 203 for the stream's HDR10 metadata (DESIGN.md §4.22).  Both bits together, either with
 *                              EXPORT_FULL_RANGE, EXPORT_BT601 or EXPORT_STRAIGHT, or on any other format are
 *                              GLAVA_B200_EINVAL.  Byte counts do not depend on them.
 *   dst[i], pitch and uv_offset are multiples of 16, pitch >= the row bytes, uv_offset (when set) >= pitch * h (planar
 *   formats: >= one chroma plane).  An unknown format or flag, odd NV12 / I420 / P010 / YUV420P10 dimensions, an odd
 *   YUV422P / YUV422P10 / UYVY width, a misaligned or short pitch (I420, YUV420P10, YUV422P, YUV422P10: not a multiple of
 *   32), a UYVY uv_offset other than 0, EXPORT_STRAIGHT with EXPORT_OVER or on a Y'CbCr format, EXPORT_OVER on a YUVA
 *   format, a null, host or other-device dst, a stream out of range, count < 1 and a renderer a failed rebuild left unbuilt
 *   are GLAVA_B200_EINVAL with nothing enqueued.  Formats 3, 9, 13 and 16 and above are unassigned.
 *   The work runs on the handle's stream (glava_b200_cuda_stream) after the latest raster pass and before the next one can
 *   overwrite a slot, so an update issued right after this call cannot change what it exports.  `after_event` (a
 *   cudaEvent_t, or NULL): the export waits for it on the device before writing the destinations — it holds back the
 *   handle's stream, and so the next raster pass, until then.  `done_event` (or NULL) is recorded after the export.
 *   Returns once the work is enqueued, without a host wait.
 *   glava_b200_export_bytes    the bytes one destination spans for `desc` on this renderer (pitch * h, UYVY included; NV12 / P010:
 *                              uv_offset + pitch * h / 2; the planar formats: pitch * h + the Cb to Cr distance + one
 *                              chroma plane; YUVA420P / YUVA444P10: pitch * h + twice the Cb to Cr distance + pitch * h),
 *                              after the same descriptor checks.
 *   glava_b200_sharded_export_frames  the same with global stream indices, dst[i] on the device of the shard that owns
 *                              streams[i]; every index and pointer is checked before any shard starts, the shards issue
 *                              concurrently, and glava_b200_sharded_sync completes the work. */
#define GLAVA_B200_EXPORT_RGBA 0
#define GLAVA_B200_EXPORT_BGRA 1
#define GLAVA_B200_EXPORT_NV12 2
#define GLAVA_B200_EXPORT_I420 4
#define GLAVA_B200_EXPORT_YUV444 5
#define GLAVA_B200_EXPORT_P010 6
#define GLAVA_B200_EXPORT_YUV420P10 7
#define GLAVA_B200_EXPORT_YUV444P10 8
#define GLAVA_B200_EXPORT_YUV422P 10
#define GLAVA_B200_EXPORT_YUV422P10 11
#define GLAVA_B200_EXPORT_UYVY 12
#define GLAVA_B200_EXPORT_YUVA420P 14
#define GLAVA_B200_EXPORT_YUVA444P10 15
#define GLAVA_B200_EXPORT_OVER 1u
#define GLAVA_B200_EXPORT_STRAIGHT 0x4u
#define GLAVA_B200_EXPORT_FULL_RANGE 0x100u
#define GLAVA_B200_EXPORT_BT601 0x200u
#define GLAVA_B200_EXPORT_PQ 0x800u
#define GLAVA_B200_EXPORT_HLG 0x1000u
typedef struct {
    int      format;            /* GLAVA_B200_EXPORT_RGBA / _BGRA / _NV12 / _I420 / _YUV444 / _P010 / _YUV420P10 /
                                   _YUV444P10 / _YUV422P / _YUV422P10 / _UYVY / _YUVA420P / _YUVA444P10 */
    uint32_t flags;             /* GLAVA_B200_EXPORT_OVER or (RGBA / BGRA) _STRAIGHT, and for the Y'CbCr formats
                                   _FULL_RANGE / _BT601, or for the 10-bit ones _PQ / _HLG */
    uint8_t  background[4];     /* R, G, B of the opaque background the composite uses; byte 3 unused */
    size_t   pitch;             /* bytes from one output row to the next (every plane; I420 / YUV420P10 / YUV422P /
                                   YUV422P10 chroma rows: pitch / 2) */
    size_t   uv_offset;         /* NV12 / P010: bytes from dst[i] to the CbCr plane, 0 = pitch * h; the planar formats:
                                   bytes from the Cb plane to the Cr plane (YUVA: and from Cr to A), 0 = one chroma
                                   plane */
} glava_b200_export;
int glava_b200_export_bytes(const glava_b200* r, const glava_b200_export* desc, size_t* bytes);
int glava_b200_export_frames(glava_b200* r, const int* streams, int count, void* const* dst,
                             const glava_b200_export* desc, void* after_event, void* done_event);

/* Scaled and cropped export (DESIGN.md §4.11), for thumbnails, encoder ladders and mosaics: glava_b200_export_frames of a
 * source rectangle shrunk to out_w x out_h, in the same single launch, reading only the rows the marks let through.
 *   glava_b200_export_scaled   the frames glava_b200_export_frames would export (same ordering, events and streams rules),
 *                              each cut to the rectangle `scale` names and downscaled by the exact area average: output
 *                              column X covers source columns [X src_w, (X + 1) src_w) / out_w, weighted by overlap, rows
 *                              likewise, and every channel is (sum of w * c + D / 2) / D with D = src_w * src_h in 64-bit
 *                              integers.  A constant image stays constant; the whole frame at its own size is exactly
 *                              glava_b200_export_frames.  RGBA / BGRA without EXPORT_OVER average the stored channels
 *                              (premultiplied under native opacity); with it, and for NV12, each source pixel is composited
 *                              first and alpha is 255.  NV12 is the export's arithmetic on the scaled image (Y per pixel,
 *                              chroma per 2x2 output block), so out_w and out_h are even; the other YUV formats likewise
 *                              apply their own arithmetic to the scaled image (out_w and out_h even for I420, P010 and
 *                              YUV420P10; out_w even for YUV422P, YUV422P10 and UYVY).
 *     dst[i]                   out_h rows of out_w * 4 bytes (RGBA / BGRA), out_w bytes (Y) or out_w uint16 (P010 and
 *                              the planar 10-bit formats' Y), `pitch` bytes apart
 *     dst_uv                   NV12 / P010: dst_uv[i] receives the out_h / 2 CbCr rows (a mosaic tile's chroma need not sit
 *                              at one offset from its luma); NULL: dst[i] + (uv_offset ? uv_offset : pitch * out_h).
 *                              Planar formats: dst_uv[i] is the Cb plane, NULL: dst[i] + pitch * out_h; the Cr plane is
 *                              uv_offset past it (0: the Cb plane's size), which lets a planar mosaic tile find its Cr rows
 *   Nothing outside each out_w x out_h rectangle and its chroma rows is written: pitch padding and neighbouring tiles keep
 *   their bytes.  dst[i], dst_uv[i], pitch and uv_offset are multiples of 16 (a mosaic tile starts at a multiple of 4 pixels
 *   in RGBA, of 16 in NV12 and YUV420P10, of 8 in YUV444P10).  Besides every refusal of glava_b200_export_frames (pitch and uv_offset measured against the
 *   output), a null `scale`, a rectangle that is empty or leaves the frame, upscaling, odd NV12 output dimensions, a
 *   misaligned, null, host or other-device dst_uv[i], and dst_uv for RGBA / BGRA / UYVY are GLAVA_B200_EINVAL with nothing
 *   enqueued.
 *   glava_b200_export_scaled_bytes   the bytes one destination spans (as glava_b200_export_bytes with out_h for h, dst_uv
 *                              NULL), after the same descriptor and rectangle checks.
 *   glava_b200_sharded_export_scaled  the same with global stream indices, dst[i] / dst_uv[i] on the device of the shard
 *                              that owns streams[i]; every entry is checked before any shard starts. */
typedef struct {
    int src_x, src_y, src_w, src_h;   /* source rectangle, top-down (row 0 = framebuffer row h - 1); src_w == src_h == 0:
                                         the whole frame */
    int out_w, out_h;                 /* 1 <= out_w <= src_w, 1 <= out_h <= src_h: downscale only */
} glava_b200_export_scale;
int glava_b200_export_scaled_bytes(const glava_b200* r, const glava_b200_export* desc, const glava_b200_export_scale* scale,
                                   size_t* bytes);
int glava_b200_export_scaled(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                             const glava_b200_export* desc, const glava_b200_export_scale* scale, void* after_event,
                             void* done_event);

/* Encoder ladder (DESIGN.md §4.13): several sizes of each frame in one launch that reads each source row about once, for an
 * ABR ladder whose rungs NVENC cannot scale itself (say 1080p, 720p and 360p NV12 beside an RGBA thumbnail).
 *   glava_b200_export_ladder   rung j of entry i gets exactly the bytes glava_b200_export_scaled(r, &streams[i], 1,
 *                              &dst[i * nrungs + j], dst_uv ? &dst_uv[i * nrungs + j] : NULL, &rungs[j].desc,
 *                              &rungs[j].scale, ...) would write at this point in call order (framebuffer ring, styles and
 *                              repeated streams included); a rung that is the whole frame at its own size is therefore
 *                              glava_b200_export_frames, bit for bit.  Formats and flags, colour flags included, may differ
 *                              between rungs, so one ladder can mix encodings.  Ordering
 *                              and events as glava_b200_export_frames: waits for `after_event` on the device, runs on the
 *                              handle's stream behind the latest pass, records `done_event`, returns without a host wait.
 *     dst                      [count][nrungs] destinations; each rung's size is glava_b200_export_scaled_bytes(r,
 *                              &rungs[j].desc, &rungs[j].scale, &n) (there is no separate byte-count call)
 *     dst_uv                   NULL, or [count][nrungs] CbCr destinations as glava_b200_export_scaled's, NULL entries for
 *                              RGBA / BGRA / UYVY rungs
 *   Nothing outside a rung's rectangle and its chroma rows is written; like glava_b200_export_scaled the call does not check
 *   whether destinations overlap.  Every refusal of glava_b200_export_scaled, checked per rung (the message names the rung),
 *   nrungs < 1 or > GLAVA_B200_LADDER_MAX, null `rungs` and a non-null dst_uv entry for an RGBA / BGRA / UYVY rung are
 *   GLAVA_B200_EINVAL with nothing enqueued.
 *   glava_b200_sharded_export_ladder  the same with global stream indices, each entry's destinations on the device of the
 *                              shard that owns streams[i]; every entry of every rung is checked before any shard starts. */
typedef struct {
    glava_b200_export       desc;     /* format, flags, background, pitch, uv_offset of this rung's destinations */
    glava_b200_export_scale scale;    /* source rectangle and output size, as glava_b200_export_scaled */
} glava_b200_export_rung;
#define GLAVA_B200_LADDER_MAX 8
int glava_b200_export_ladder(glava_b200* r, const int* streams, int count, const glava_b200_export_rung* rungs, int nrungs,
                             void* const* dst, void* const* dst_uv, void* after_event, void* done_event);

/* Overlay onto the caller's images (DESIGN.md §4.12), for audiograms, music channels and compositing over video: the frames
 * drawn over a picture the caller holds in DEVICE memory, in place, in one launch that touches only what the frame covers.
 *   glava_b200_overlay_frames  composites the current frame of streams[i] — what glava_b200_export_frames would export
 *                              (same ordering, events and streams rules), top-down — onto the w x h rectangle at dst[i]:
 *     dst[i]                   the rectangle's top-left pixel (RGBA / BGRA: 4-byte pixels) or Y byte (NV12), `pitch`
 *                              bytes per row; the caller's image around it is never touched
 *     dst_uv                   NV12: dst_uv[i] is the rectangle's first CbCr byte; NULL: dst[i] + (uv_offset ? uv_offset :
 *                              pitch * h), as glava_b200_export_scaled
 *     desc                     format and pitch (and uv_offset) as the export; background is unused; flags 0, or for
 *                              NV12 the colour flags EXPORT_FULL_RANGE / EXPORT_BT601, the picture's encoding: the blend
 *                              takes that set's coefficients and offsets (full range: T = 0 a + (255 - a) Y_D for Y)
 *   Under setopacity "native" (premultiply_alpha) the stored premultiplied pixel goes "over" the caller's pixel D, as
 *   GLava's window goes over the desktop: RGBA / BGRA C = min(255, c + mul_norm8(D, 255 - a)) in all four channels (D
 *   opaque or premultiplied); NV12 blends in Y'CbCr without a trip through RGB, Y = clamp((Y_R r + Y_G g + Y_B b +
 *   floor((T 2^16 + 127) / 255) + 2^15) >> 16), T = 16 a + (255 - a) Y_D, and Cb / Cr likewise with T = 128 a + (255 - a)
 *   Cb_D (Cr_D) from the (s + 2) >> 2 average of the 2x2 block's stored pixels, alpha included (export_core.h).  A zero
 *   pixel leaves D exactly as it was, and rows the dirty-row marks skip and all-zero quads are neither read nor written.
 *   An opaque pixel gives exactly glava_b200_export_frames' bytes.  Under any other opacity GLava's window is opaque: the
 *   rectangle gets exactly what glava_b200_export_frames writes (RGBA / BGRA with EXPORT_OVER, or NV12).
 *   The overlay takes RGBA, BGRA and NV12; I420, YUV444, P010, YUV420P10, YUV444P10, YUV422P, YUV422P10 and UYVY are
 *   refused by name (decoded
 *   pictures in those formats, with per-plane pointers and pitches, go to glava_b200_overlay_planes below).
 *   Besides the refusals of glava_b200_export_scaled that apply (format, pitch, uv_offset, alignment, null / host /
 *   other-device dst or dst_uv, dst_uv for RGBA / BGRA, odd NV12 frames, stream range, count < 1, an unbuilt renderer),
 *   any other flag, a rectangle that meets the renderer's framebuffer array and two rectangles of one call that overlap (luma
 *   and chroma planes included: each entry reads and writes its bytes; layers go in separate calls) are GLAVA_B200_EINVAL
 *   with nothing enqueued.
 *   glava_b200_sharded_overlay_frames  the same with global stream indices, dst[i] / dst_uv[i] on the device of the shard
 *                              that owns streams[i]; every entry, the overlap of the whole list and every shard's
 *                              framebuffer are checked before any shard starts. */
int glava_b200_overlay_frames(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                              const glava_b200_export* desc, void* after_event, void* done_event);

/* Overlay onto decoded pictures (DESIGN.md §4.17, §4.18): what a decoder or ffmpeg hands over — NV12, I420, YUV444, P010,
 * YUV420P10, YUV444P10, YUV422P, YUV422P10 or UYVY, each plane at its own pointer, luma and chroma rows at their own
 * pitches.
 *   glava_b200_overlay_planes  composites the current frame of streams[i] onto the w x h rectangle of pics[i], exactly as
 *                              glava_b200_overlay_frames does onto NV12 (same ordering, events, streams and opacity rules;
 *                              NV12 runs its item body), top-down at the rectangle's origin:
 *     pics[i].plane[0]         the rectangle's first Y sample (UYVY: its first Cb byte), `pitch` bytes per row
 *     pics[i].plane[1]         NV12 / P010: its first CbCr pair; the planar formats: its first Cb sample; NULL for UYVY
 *     pics[i].plane[2]         the planar formats: its first Cr sample; NULL for NV12, P010 and UYVY
 *     desc                     format, flags (0, or EXPORT_FULL_RANGE / EXPORT_BT601: the picture's encoding), the luma
 *                              pitch and one chroma pitch for every chroma plane (UYVY: 0); 4:2:0 chroma is w/2 x h/2,
 *                              4:2:2 chroma w/2 x h
 *   10-bit samples hold their code as v >> 6 (P010) or v & 1023 (YUV420P10, YUV444P10).  Under native opacity the blend is
 *   overlay_frames' NV12 blend (I420: bit for bit NV12 deinterleaved; YUV444: chroma per pixel), and at 10 bits the same
 *   fraction at 10 bits with 4:2:0 chroma from the block's exact sums, as P010's export (export_core.h); 4:2:2 chroma is
 *   the 4:2:0 blend of the block whose two rows are the pixel pair.  A blended 10-bit
 *   sample is written with its other bits zero; a sample no non-zero pixel covers (a luma sample under a zero pixel, a chroma
 *   sample whose pixel or 2x2 block is all zero) keeps all 16 bits, and rows the marks skip and all-zero quads are neither
 *   read nor written.  Under any other opacity every sample of the rectangle gets glava_b200_export_frames' bytes.
 *   HDR pictures (DESIGN.md §4.22): EXPORT_PQ or EXPORT_HLG on P010, YUV420P10, YUV444P10 or YUV422P10 says the picture is
 *   BT.2020 PQ / HLG limited range; the blend then takes each pixel's straight colour S in the HDR export's arithmetic, Y =
 *   round((a Y_f(S) + (255 - a) Y_D) / 255) and chroma round(512 + sum a_i (C_f(S_i) - 512) / (255 n) + (1 - A / (255 n))
 *   (C_D - 512)) over the n pixels of a block / pair / pixel, so graphics land at 203 cd/m^2, an opaque pixel gives the HDR
 *   export's codes and zero pixels keep every bit.  Either bit on another format, both, or with EXPORT_FULL_RANGE /
 *   EXPORT_BT601 is GLAVA_B200_EINVAL; glava_b200_overlay_frames takes neither.
 *   GLAVA_B200_EINVAL, with nothing enqueued, for: a null argument, count < 1, an unbuilt renderer; RGBA, BGRA (those go to
 *   glava_b200_overlay_frames) or an unknown format; any other flag; odd w or h for the 4:2:0 formats, odd w for the 4:2:2
 *   ones; a pitch or chroma_pitch that is not a multiple of 16 or below the plane's row bytes (luma w, 2w at 10 bits and
 *   for UYVY; chroma w for NV12, YUV444, YUV420P10 and YUV422P10, w/2 for I420 and YUV422P, 2w for P010 and YUV444P10); a
 *   UYVY chroma_pitch other than 0; a plane pointer that is null, not 16-byte aligned, not device memory or on another
 *   device; a non-null plane[2] for NV12 or P010, a non-null plane[1] or plane[2] for UYVY; a stream out of range; a plane rectangle
 *   that meets the renderer's framebuffer array; two plane rectangles of the call that overlap (every pair: across
 *   entries, luma against chroma, Cb against Cr).
 *   glava_b200_sharded_overlay_planes  the same with global stream indices, each picture on the device of the shard that
 *                              owns streams[i]; every entry, the overlap of the whole list and every shard's framebuffer are
 *                              checked before any shard starts. */
typedef struct { void* plane[3]; } glava_b200_picture;
typedef struct {
    int      format;        /* GLAVA_B200_EXPORT_NV12, _I420, _YUV444, _P010, _YUV420P10, _YUV444P10, _YUV422P,
                               _YUV422P10, _UYVY */
    uint32_t flags;         /* 0, or GLAVA_B200_EXPORT_FULL_RANGE / GLAVA_B200_EXPORT_BT601, or (10-bit formats)
                               GLAVA_B200_EXPORT_PQ / GLAVA_B200_EXPORT_HLG */
    size_t   pitch;         /* bytes between luma rows */
    size_t   chroma_pitch;  /* bytes between rows of every chroma plane */
} glava_b200_overlay_planes_desc;
int glava_b200_overlay_planes(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                              const glava_b200_overlay_planes_desc* desc, void* after_event, void* done_event);

/* Overlay at a per-entry opacity (DESIGN.md §4.20), for fading a visualiser in and out and running it translucent over video:
 *   glava_b200_overlay_frames_opacity / glava_b200_overlay_planes_opacity  the plain calls with one more argument,
 *     opacity                  [count] opacities K, 0..255, of the entries (read during the call, as streams); NULL: all 255
 *   Entry i composites a pixel scaled by K_i / 255 in all four channels with the blend path's unorm8 product (mul_norm8, so
 *   premultiplied colour stays at or below alpha) through the format's native blend.  Under setopacity "native" the pixel
 *   is the stored premultiplied one; under any other opacity GLava's window is opaque and it is the stored colour with
 *   alpha 255, which at K = 255 gives exactly the plain call's bytes.  K = 255 is the plain call bit for bit, K = 0 leaves
 *   the picture untouched; against the float64 composite c K / 255 + D (1 - a K / 255^2) the result stays within the
 *   bounds DESIGN.md §4.20 records per format and encoding.  Every refusal of the plain call applies unchanged, to every
 *   entry (K = 0 ones included), and names the _opacity call.  A list whose K are all 255 (or NULL) runs the plain
 *   kernel; K = 0 entries are left out of the device list, and a list of only those enqueues no kernel (the stream still
 *   waits for after_event and records done_event).
 *   glava_b200_sharded_overlay_frames_opacity / glava_b200_sharded_overlay_planes_opacity  the sharded forms, opacity[i]
 *                              travelling with streams[i]. */
int glava_b200_overlay_frames_opacity(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                                      const glava_b200_export* desc, const uint8_t* opacity /* [count], NULL = all 255 */,
                                      void* after_event, void* done_event);
int glava_b200_overlay_planes_opacity(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                                      const glava_b200_overlay_planes_desc* desc, const uint8_t* opacity /* [count], NULL = all 255 */,
                                      void* after_event, void* done_event);

/* Overlay a downscaled, cropped frame (DESIGN.md §4.21), for picture-in-picture and for the same visualiser on every rendition
 * of an overlaid video:
 *   glava_b200_overlay_scaled  streams, pics and desc as glava_b200_overlay_planes, with the formats RGBA and BGRA added (only
 *                              plane[0], chroma_pitch 0, flags 0); scale as glava_b200_export_scaled (a source rectangle, top-down,
 *                              all zero = the whole frame; out_w x out_h, downscale only); opacity as
 *                              glava_b200_overlay_planes_opacity; after_event / done_event as glava_b200_export_frames.
 *   The rectangle in pics[i] is out_w x out_h.  Entry i leaves there exactly what glava_b200_overlay_planes_opacity (RGBA /
 *   BGRA: glava_b200_overlay_frames_opacity) would leave with opacity[i] if the stream's frame were S_i, the out_w x out_h
 *   RGBA image glava_b200_export_scaled of streams[i] with this scale writes at this point in call order: under setopacity
 *   "native" with flags 0 (the premultiplied exact area average), under any other opacity with EXPORT_OVER (each pixel made
 *   opaque before the average).  Ordered on the raster stream as the other overlays; streams may repeat.  Hence, bit for bit:
 *   the whole frame at its own size is glava_b200_overlay_planes_opacity / _overlay_frames_opacity (whose kernels it runs);
 *   under any other opacity at K = 255 the rectangle holds glava_b200_export_scaled's bytes of the format and encoding
 *   (RGBA / BGRA: with EXPORT_OVER); a frame of zero pixels under native opacity, and K = 0 in any mode, leave the picture
 *   untouched (an all-zero quad of S_i is neither read nor written, and a 10-bit sample no non-zero pixel covers keeps all
 *   16 bits).  K = 0 entries are left out of the device list; a list of only those enqueues no kernel, but the stream
 *   still waits for after_event and records done_event.
 *   GLAVA_B200_EINVAL, with nothing enqueued and the message naming the call, for: every refusal of glava_b200_overlay_planes
 *   measured against out_w x out_h (parity, pitches, plane pointers, stream range, count, an unbuilt renderer, overlap with
 *   the framebuffer array or between any two plane rectangles of the call); a null scale, a source rectangle that is empty or
 *   leaves the frame, an output larger than the source; EXPORT_STRAIGHT, EXPORT_OVER or any other flag (RGBA / BGRA: any
 *   flag), the YUVA formats; for RGBA / BGRA a non-null plane[1] or plane[2] or a non-zero chroma_pitch.
 *   glava_b200_sharded_overlay_scaled  the same with global stream indices, each picture on the device of the shard that
 *                              owns streams[i]; every entry and the overlap of the whole list are checked before any shard starts. */
int glava_b200_overlay_scaled(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                              const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale,
                              const uint8_t* opacity /* [count], NULL = all 255 */, void* after_event, void* done_event);

/* ---- one handle for a batch spread over several GPUs of a node (csrc/sharded.cpp) -------------------------------------
 * The streams of a batch are independent (one GLava process each, in the reference), so the batch is cut into contiguous
 * blocks, one per device — glava_b200_shard_range: counts differ by at most one — and nothing crosses between devices (no
 * collective, NCCL unused).  One worker thread per device, pinned to the device's NUMA node; every call below is issued
 * on all shards concurrently.  lb / rb / chunks / modified / textures are indexed by GLOBAL stream, [batch][...].
 *   device_mask: bit d = CUDA device d takes a shard (0 = every visible device).  _devices: explicit ordinals (an
 *   ordinal may repeat: several shards on one device).  Error behaviour as everywhere: 0 / negative code + abort hook;
 *   the message names the failing device and its stream block. */
typedef struct glava_b200_sharded glava_b200_sharded;
int  glava_b200_device_count(void);
int  glava_b200_shard_range(int batch, int shards, int k, int* first_stream, int* count);
glava_b200_sharded* glava_b200_new_sharded(const glava_b200_params* params, int batch, uint64_t device_mask);
glava_b200_sharded* glava_b200_new_sharded_devices(const glava_b200_params* params, int batch, const int* devices, int n);
void glava_b200_sharded_destroy(glava_b200_sharded* s);
int  glava_b200_sharded_shards(const glava_b200_sharded* s);
int  glava_b200_sharded_batch(const glava_b200_sharded* s);
glava_b200* glava_b200_sharded_shard(const glava_b200_sharded* s, int k, int* device, int* first_stream, int* count);
int  glava_b200_sharded_update(glava_b200_sharded* s, const float* lb, const float* rb, size_t bsz, const uint8_t* modified /* NULL: all */);
int  glava_b200_sharded_rerender(glava_b200_sharded* s);                                  /* rd_update(modified = false) */
int  glava_b200_sharded_ingest_fifo(glava_b200_sharded* s, const int16_t* chunks, int frames);   /* ingest + update on the rings */
int  glava_b200_sharded_sync(glava_b200_sharded* s);
int  glava_b200_sharded_readback(glava_b200_sharded* s, int stream, uint8_t* rgba);
const void* glava_b200_sharded_frame_device(glava_b200_sharded* s, int stream, int* device);
int  glava_b200_sharded_textures(glava_b200_sharded* s, uint16_t* out_l, uint16_t* out_r);
int  glava_b200_sharded_export_frames(glava_b200_sharded* s, const int* streams, int count, void* const* dst,
                                      const glava_b200_export* desc);   /* global indices; see glava_b200_export_frames */
int  glava_b200_sharded_export_scaled(glava_b200_sharded* s, const int* streams, int count, void* const* dst,
                                      void* const* dst_uv, const glava_b200_export* desc,
                                      const glava_b200_export_scale* scale);   /* global indices; see glava_b200_export_scaled */
int  glava_b200_sharded_overlay_frames(glava_b200_sharded* s, const int* streams, int count, void* const* dst,
                                       void* const* dst_uv, const glava_b200_export* desc);   /* see glava_b200_overlay_frames */
int  glava_b200_sharded_overlay_planes(glava_b200_sharded* s, const int* streams, int count, const glava_b200_picture* pics,
                                       const glava_b200_overlay_planes_desc* desc);   /* see glava_b200_overlay_planes */
int  glava_b200_sharded_overlay_frames_opacity(glava_b200_sharded* s, const int* streams, int count, void* const* dst,
                                               void* const* dst_uv, const glava_b200_export* desc,
                                               const uint8_t* opacity);   /* see glava_b200_overlay_frames_opacity */
int  glava_b200_sharded_overlay_planes_opacity(glava_b200_sharded* s, const int* streams, int count, const glava_b200_picture* pics,
                                               const glava_b200_overlay_planes_desc* desc,
                                               const uint8_t* opacity);   /* see glava_b200_overlay_planes_opacity */
int  glava_b200_sharded_overlay_scaled(glava_b200_sharded* s, const int* streams, int count, const glava_b200_picture* pics,
                                       const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale,
                                       const uint8_t* opacity);   /* see glava_b200_overlay_scaled */
int  glava_b200_sharded_export_ladder(glava_b200_sharded* s, const int* streams, int count,
                                      const glava_b200_export_rung* rungs, int nrungs, void* const* dst,
                                      void* const* dst_uv);   /* global indices; see glava_b200_export_ladder */

/* ---- lifetime of individual streams: reset, save and load (DESIGN.md §4.8) -------------------------------------------
 * A stream's state is what its next update reads besides its new audio: gravity store and average ring, the latest
 * spectrum, the texture the next raster reads, the pre-smoothing texture and the device FIFO ring.
 *   glava_b200_stream_state_bytes  bytes of one stream's blob for renderers created with `p`:
 *                                  GLAVA_B200_STATE_HEADER_BYTES + chans * ((1 + F) * n * esz + 8 * n + 4 * setbufsize),
 *                                  n = setbufsize / setbufscale, F = setavgframes, esz = 2 under setaccelfft (pipeline B) and
 *                                  4 otherwise (an appended "smooth" transform clears setaccelfft), chans = 1 for wave, else 2.
 *                                  0 (with the error set) when keyframe interpolation is active or `p` is invalid.
 *   glava_b200_reset_streams       every stream with mask[s] != 0 becomes stream 0 of a newly created renderer: from its next
 *                                  update on it renders what a fresh batch-1 renderer fed the same calls renders.  Its
 *                                  framebuffer slot keeps the old frame until then.  Does not wait for the device.
 *   glava_b200_save_streams        writes the state of streams[0 .. count) into `blobs` (HOST, count * bytes; pinned memory
 *                                  from glava_b200_host_alloc copies at the PCIe rate).  Returns once the blobs are complete.
 *   glava_b200_load_streams        puts blobs saved from a renderer with the same effective parameters (fb_slots aside) into
 *                                  streams[0 .. count) of this one, whatever its batch, device, update count or ring cursors:
 *                                  each slot then continues exactly as the saved stream would have.  Returns once the blobs
 *                                  have been consumed, like glava_b200_update; does not wait for earlier updates.
 * All three are ordered with the handle's updates like any other call.  GLAVA_B200_EINVAL, with nothing touched, for
 * stream indices out of range or repeated, a blob of other parameters, magic, version or size, and while keyframe
 * interpolation is active (the keyframe rotation belongs to the renderer, as for uneven masks).  The format is not
 * stable across library versions: the version field rejects a mismatch.
 * The sharded forms take global stream indices (mask: [batch] in global order); a stream moves between shards by a
 * save on one and a load on the other. */
#define GLAVA_B200_STATE_HEADER_BYTES 4096
size_t glava_b200_stream_state_bytes(const glava_b200_params* p);
int glava_b200_reset_streams(glava_b200* r, const uint8_t* mask /* [batch], non-zero = reset */);
int glava_b200_save_streams(glava_b200* r, const int* streams, int count, void* blobs /* HOST, count * bytes */);
int glava_b200_load_streams(glava_b200* r, const int* streams, int count, const void* blobs);
int glava_b200_sharded_reset_streams(glava_b200_sharded* s, const uint8_t* mask /* [batch], global order */);
int glava_b200_sharded_save_streams(glava_b200_sharded* s, const int* streams, int count, void* blobs);
int glava_b200_sharded_load_streams(glava_b200_sharded* s, const int* streams, int count, const void* blobs);

/* ---- per-stream looks (DESIGN.md §4.9) --------------------------------------------------------------------------------
 *   glava_b200_style_params       `base` with the style `s` applied (see glava_b200_stream_style): what a batch-1 renderer
 *                                 needs to render what a stream of that style renders.  GLAVA_B200_EINVAL for a style
 *                                 the module cannot take or parameters that fail validation.
 *   glava_b200_set_stream_styles  gives streams[i] the style styles[i]; a style with set == 0 returns the stream to the
 *                                 renderer's own look.  From the next raster pass on (a modified = 0 update re-rasters the
 *                                 old spectrum in the new look), stream s renders, byte for byte, what a batch-1 renderer
 *                                 created with glava_b200_style_params(current parameters, style of s) renders when fed
 *                                 the same calls.  Textures and spectra do not depend on styles.  Out-of-range or repeated
 *                                 indices and any invalid style are GLAVA_B200_EINVAL with nothing changed.  The tables are
 *                                 rebuilt as on glava_b200_reconfigure, with its out-of-memory behaviour.
 *   glava_b200_get_stream_styles  the styles of streams[0 .. count), as set (set == 0: none)
 * Styles belong to the stream slot: glava_b200_reconfigure and glava_b200_sizereq keep them (an unstyled field follows the
 * new parameters; a reconfigure that would make a style invalid is refused), reset / save / load of streams leave them
 * alone.  The sharded forms take global stream indices; they check every index and style before any shard starts, but a
 * shard whose table rebuild then fails (out of memory) is left as glava_b200_set_stream_styles leaves it, while the shards
 * that succeeded keep their new styles: after such a failure, read the styles back or set them again. */
int glava_b200_style_params(const glava_b200_params* base, const glava_b200_stream_style* s, glava_b200_params* out);
/* "#rrggbb" / "#rrggbbaa" -> RGBA floats, rounded as a `--pipe` bind of that text is (GLAVA_B200_EINVAL: not such a colour) */
int glava_b200_parse_hex_color(const char* text, float rgba[4]);
int glava_b200_set_stream_styles(glava_b200* r, const int* streams, int count, const glava_b200_stream_style* styles);
int glava_b200_get_stream_styles(const glava_b200* r, const int* streams, int count, glava_b200_stream_style* out);
int glava_b200_sharded_set_stream_styles(glava_b200_sharded* s, const int* streams, int count, const glava_b200_stream_style* styles);
int glava_b200_sharded_get_stream_styles(const glava_b200_sharded* s, const int* streams, int count, glava_b200_stream_style* out);

/* Stage-wise entry points (used by the parity tests; same kernels as the fused path). */
int glava_b200_smooth_pass(glava_b200* r, const uint16_t* in, uint16_t* out, int count);      /* K5 on HOST [count][n] */
int glava_b200_raster_textures(glava_b200* r, const uint16_t* tex_l, const uint16_t* tex_r);  /* HOST [batch][n] -> raster */
int glava_b200_transform_smooth(glava_b200* r, float* planes, int count);                     /* transform_smooth in place on HOST [count][n] */

/* Kernel launch counters since creation (bench.py `gpu_launches`). */
uint64_t glava_b200_launch_count(const glava_b200* r);

/* Per-kernel device timing: when enabled, CUDA events are recorded on the handle's stream around
 * the spectrum kernel and the raster kernel of every update; glava_b200_kernel_times() synchronises
 * and returns the summed durations (ms) and launch counts since timing was (re-)enabled. */
int glava_b200_set_timing(glava_b200* r, int enable);
int glava_b200_kernel_times(glava_b200* r, double* spectrum_ms, int* spectrum_launches,
                            double* raster_ms, int* raster_launches);
/* development aid: [start, end] ms of every timed launch relative to the first one (spectrum pairs, then raster pairs) */
int glava_b200_timeline(glava_b200* r, double* out, int cap_pairs, int* n_spec, int* n_ras);

/* ---- audio plug-in ABI kept verbatim from the reference (fifo.h:9-26) so a GLava audio
 * backend can feed this renderer: see INTEGRATION.md. ---- */

const char* glava_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GLAVA_B200_H */
