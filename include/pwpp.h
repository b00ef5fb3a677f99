/*
 * pwpp.h — thin C-ABI of the H100 ground-segmentation engine (libpwpp_b200.so).
 *
 * This is the drop-in boundary for ONE path of url-kaist/patchwork-plusplus:
 * patchwork::PatchWorkpp::estimateGround() and the getters that read its result.
 * Everything above this header (the C++ class `patchwork::PatchWorkpp` in
 * include/patchwork/patchworkpp.h and the Python module `pypatchworkpp`) is glue.
 * No torch / Eigen / STL types cross this boundary: plain pointers, sizes, PODs.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the
 * reference checkout, commit b608129a):
 *   H  = cpp/patchworkpp/include/patchwork/patchworkpp.h
 *   S  = cpp/patchworkpp/src/patchworkpp.cpp
 *   PB = python/patchworkpp/pybinding.cpp
 *
 * Model: a `pwpp_ctx` owns `num_streams` independent sensor streams. One stream is what
 * the reference calls one PatchWorkpp instance (H:114-235): it carries the temporal state
 * (adaptive elevation/flatness thresholds, their histories, the adaptive sensor height —
 * S:338-375) from frame to frame. pwpp_estimate_host / pwpp_estimate_device process ONE frame
 * for each of the first `nframes` streams, all on the GPU, in a single launch sequence. The
 * *_streams variants take a stream table instead: frame f of the call belongs to stream
 * streams[f], any subset of the streams in any order, a stream possibly several times (its
 * frames then run in call order, see "Stream table" below). The reference class maps to a ctx
 * with num_streams == 1.
 *
 * Indexing rule: everything a call PRODUCES is indexed by the frame's position f in the call
 * (counts, index lists, xyz, centers, normals, patch records, bin ids, pwpp_device_results,
 * pwpp_host_results); the temporal STATE is indexed by stream id (pwpp_get_state, pwpp_height,
 * pwpp_copy_history, pwpp_export_state / pwpp_import_state, pwpp_reset_stream). With the
 * identity table of pwpp_estimate_host / pwpp_estimate_device the two coincide. The PARAMETERS a frame
 * runs with are those of its stream's set (pwpp_create_sets; one set for a ctx from pwpp_create): results
 * by call position, state by stream id, parameters by the stream's set.
 *
 * All functions returning int return PWPP_OK (0) or a negative pwpp_status; the message
 * for the last failure on the calling thread is available from pwpp_last_error().
 * There is NO CPU fallback: creating a ctx without a usable CUDA device fails loudly.
 */
#ifndef PWPP_H_
#define PWPP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PWPP_ABI_VERSION 1
#define PWPP_NUM_ZONES 4            /* H:127-134 hard-wires 4 zones via .at(0..3)          */
#define PWPP_MAX_RINGS_OF_INTEREST 4 /* H:174-175: update_flatness_[4], update_elevation_[4] */
#define PWPP_MAX_PARAM_SETS 8       /* parameter sets of one ctx (pwpp_create_sets) */

typedef enum pwpp_status {
  PWPP_OK = 0,
  PWPP_ERR_INVALID_ARG = -1,
  PWPP_ERR_CUDA = -2,
  PWPP_ERR_NO_DEVICE = -3,
  PWPP_ERR_UNSUPPORTED = -4,
  PWPP_ERR_CAPACITY = -5
} pwpp_status;

/* POD mirror of patchwork::Params (H:42-112); field names, meaning and defaults identical.
 * The std::vector fields become fixed [4] arrays (the reference only ever reads 4 entries).
 * `intensity_thr` is bound in Python (PB:37) but never read by the algorithm; kept for shape. */
typedef struct pwpp_params {
  int32_t verbose;                 /* H:44  (bool) */
  int32_t enable_RNR;              /* H:45  */
  int32_t enable_RVPF;             /* H:46  */
  int32_t enable_TGR;              /* H:47  */
  int32_t num_iter;                /* H:49  default 3  */
  int32_t num_lpr;                 /* H:50  default 20 */
  int32_t num_min_pts;             /* H:51  default 10 */
  int32_t num_zones;               /* H:52  must be 4  */
  int32_t num_rings_of_interest;   /* H:53  default 4, must be <= 4 */
  int32_t max_flatness_storage;    /* H:72  default 1000 */
  int32_t max_elevation_storage;   /* H:73  default 1000 */
  int32_t _pad0;
  double RNR_ver_angle_thr;        /* H:55  default -15.0 */
  double RNR_intensity_thr;        /* H:56  default 0.2   */
  double sensor_height;            /* H:58  default 1.723 (adaptive, S:348) */
  double th_seeds;                 /* H:59  default 0.125 */
  double th_dist;                  /* H:60  default 0.125 */
  double th_seeds_v;               /* H:61  default 0.25  */
  double th_dist_v;                /* H:62  default 0.1   */
  double max_range;                /* H:63  default 80.0  */
  double min_range;                /* H:64  default 2.7   */
  double uprightness_thr;          /* H:65  default 0.707 */
  double adaptive_seed_selection_margin; /* H:66 default -1.2 */
  double intensity_thr;            /* H:67  unused by the algorithm */
  int32_t num_sectors_each_zone[PWPP_NUM_ZONES]; /* H:69 default {16,32,54,32} */
  int32_t num_rings_each_zone[PWPP_NUM_ZONES];   /* H:70 default {2,4,4,4}     */
  double elevation_thr[PWPP_MAX_RINGS_OF_INTEREST]; /* H:75 default {0,0,0,0} (adaptive) */
  double flatness_thr[PWPP_MAX_RINGS_OF_INTEREST];  /* H:76 default {0,0,0,0} (adaptive) */
} pwpp_params;

/* Fills *p with the reference defaults (H:79-111). */
void pwpp_params_default(pwpp_params* p);

/* Temporal state of one stream — exactly the members the reference mutates between frames
 * (S:347-350, S:368, S:255-256, S:354-355, S:372-373). Used by tests and for
 * checkpoint / stream migration between GPUs. Histories hold at most
 * max_*_storage + (max bins per ring) entries; `hist_cap` is the row capacity in doubles.
 * BOUND (defined deviation, DESIGN.md section 3): a history row keeps its newest
 * hist_cap = max(max_elevation_storage, max_flatness_storage) + 4 * (max sectors of a zone) + 64 samples. The reference's
 * vectors are unbounded while ring 0 holds <= 1 flatness samples (the `break` of S:363-364 then skips the trimming of rings
 * 1..3); after more than hist_cap accepted patches of one ring in that state the reference averages over the whole history, this
 * library over the newest hist_cap samples. The state blob of pwpp_export_state depends on hist_cap (checked on import).
 * NO-PLANE PATCHES (defined deviation): a patch all of whose seed sets are empty has no plane of its own; the reference
 * (S:49) then partitions it with the normal_/d_ left behind by the previous estimate_plane call. Here all points of such a patch
 * are non-ground and A-GLE sees the carried mean / normal / singular values (pwpp_bin_result.verdict == -1 marks the patch). */
typedef struct pwpp_state {
  double sensor_height;
  double elevation_thr[PWPP_MAX_RINGS_OF_INTEREST];
  double flatness_thr[PWPP_MAX_RINGS_OF_INTEREST];
  int32_t n_elevation[PWPP_MAX_RINGS_OF_INTEREST];
  int32_t n_flatness[PWPP_MAX_RINGS_OF_INTEREST];
} pwpp_state;

typedef struct pwpp_ctx pwpp_ctx;

/* ---- lifetime -------------------------------------------------------------------------- */

/* Replaces PatchWorkpp::PatchWorkpp(Params) (H:120-150): builds the concentric-zone geometry
 * (H:122-134) and `num_streams` fresh stream states on CUDA device `device`.
 * `max_points_per_frame` sizes the per-frame device buffers (frames may be smaller);
 * capacity grows on demand if a later call exceeds it. */
int pwpp_create(const pwpp_params* params, int device, int num_streams,
                int64_t max_points_per_frame, pwpp_ctx** out);

/* Several parameter sets in one ctx: stream s runs with sets[stream_set[s]] for its whole life, exactly like a
 * reference instance constructed with those Params (H:120), and one call may mix streams of any sets. Per-frame
 * results follow the frame's set: pwpp_copy_bin_results writes that set's nbins records, pwpp_copy_bin_ids uses its
 * pseudo-bin ids (nbins, nbins + 1), centers / normals / patch counts cover its bins. State follows the stream's set:
 * reset restores the set's sensor_height / elevation_thr / flatness_thr, the history bound (hist_cap, see pwpp_state)
 * is the set's own, and a stream's state blob is the one a one-set ctx with that set produces (importable either way).
 * Every set goes through the checks of pwpp_create; num_sets must be in [1, PWPP_MAX_PARAM_SETS] and stream_set a
 * non-NULL array of num_streams ids in [0, num_sets). A failure returns PWPP_ERR_INVALID_ARG or PWPP_ERR_UNSUPPORTED
 * (the message names the set) before anything is allocated. pwpp_create is this with one set. */
int pwpp_create_sets(const pwpp_params* sets, int num_sets, const int32_t* stream_set, int device, int num_streams,
                     int64_t max_points_per_frame, pwpp_ctx** out);
void pwpp_destroy(pwpp_ctx* ctx);

const char* pwpp_last_error(void);
int pwpp_abi_version(void);
/* Number of polar bins of the configured concentric-zone model (504 with defaults). With several parameter sets: the
 * largest bin count of the sets (a pwpp_copy_bin_results buffer of that size fits any frame). */
int pwpp_num_bins(const pwpp_ctx* ctx);
/* Bin count of stream s's parameter set, and the set id of stream s (negative status for a bad s). */
int pwpp_stream_num_bins(const pwpp_ctx* ctx, int s);
int pwpp_stream_set(const pwpp_ctx* ctx, int s);

/* ---- the hot path ---------------------------------------------------------------------- */

/* Replaces PatchWorkpp::estimateGround(Eigen::MatrixXf) (H:152, S:151-336) for HOST buffers.
 * Frame f (0 <= f < nframes <= num_streams) is read from pts[f]: n[f] points of `cols`
 * (3 or 4) floats; element (i,c) is at pts[f][i*row_stride + c*col_stride] (so both numpy
 * C-order N x C and Eigen column-major N x C are accepted without a caller-side copy).
 * cols == 3 disables RNR for that call exactly like S:379-382.
 * Copies host->device through pinned staging, runs all stages on the GPU, and leaves the
 * results on the device; the copy_* getters below fetch them. The caller's buffers are
 * never modified (the reference mutates only its by-value copy, S:394). */
int pwpp_estimate_host(pwpp_ctx* ctx, int nframes, const float* const* pts, const int64_t* n,
                       int cols, int64_t row_stride, int64_t col_stride);

/* Same path for DEVICE-resident input (used by the benchmark's device-resident leg and by
 * GPU pipelines): `d_pts` is a device pointer to packed float4 {x,y,z,intensity} points of
 * all frames back to back; frame f occupies [h_offsets[f], h_offsets[f+1]) (host array of
 * nframes+1 int64). `has_intensity` == 0 behaves like cols == 3. `cuda_stream` is a
 * cudaStream_t (may be NULL = the ctx's own stream). Asynchronous w.r.t. the host: results
 * are ready after pwpp_synchronize() (the copy_* getters synchronize themselves). */
int pwpp_estimate_device(pwpp_ctx* ctx, int nframes, const void* d_pts,
                         const int64_t* h_offsets, int has_intensity, void* cuda_stream);

/* The same for packed N x 3 rows {x, y, z} resident on the device (no intensity: RNR is skipped like for N x 3 host input,
 * S:379-382): the rows are padded to the kernels' 16-byte points by a device-side copy into the ctx's input buffer. */
int pwpp_estimate_device_xyz(pwpp_ctx* ctx, int nframes, const void* d_xyz, const int64_t* h_offsets, void* cuda_stream);

/* Stream table: the same two paths with frame f of the call belonging to stream streams[f]
 * (0 <= streams[f] < num_streams; 1 <= nframes <= 65535, nframes may exceed num_streams).
 *   - Any subset of the streams, in any order. Streams the call does not name keep their state untouched.
 *   - A stream may appear several times: its frames are processed in call order, each one sees the state the
 *     previous one left (exactly as in separate calls). The call is split into maximal runs of consecutive
 *     frames with pairwise distinct streams; each run is one launch sequence over its frames, and stream
 *     order serialises the runs. In pwpp_estimate_host the launch ranges are its pipeline chunks cut at the
 *     run boundaries, so the upload of later frames still overlaps the kernels of earlier ones.
 *   - Results are indexed by call position f, state by stream id (the indexing rule above).
 *   - A NULL table, an id out of range or nframes outside [1, 65535] returns PWPP_ERR_INVALID_ARG before anything
 *     is launched: no stream's state changes.
 * pwpp_estimate_host / pwpp_estimate_device are these with the identity table streams[f] = f. */
int pwpp_estimate_host_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float* const* pts, const int64_t* n,
                               int cols, int64_t row_stride, int64_t col_stride);
int pwpp_estimate_device_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* d_pts, const int64_t* h_offsets,
                                 int has_intensity, void* cuda_stream);

/* ---- sensor point records of any PointCloud2 layout ------------------------------------------------------------------
 * A frame may also be handed over as the sensor driver published it: n[f] records of layouts[f].point_step bytes starting at
 * frames[f] (any alignment, any step: 22, 13 and 17 are as valid as 16), with the byte offset and datatype of the x, y, z and
 * intensity fields inside a record (sensor_msgs/PointField). One kernel unpacks every frame of a launch range on the GPU into
 * the ctx's own float4 input buffer; everything after that is the path of pwpp_estimate_host / pwpp_estimate_device.
 *   - Every frame carries its own layout, so one call may mix sensors of different drivers. Results by call position, state
 *     by stream id, parameters by the stream's set, layout by the frame. The stream table (required, non-NULL) works exactly
 *     as for the *_streams entry points: same checks, same error codes, same run splitting.
 *   - Fields are converted to float by value with round-to-nearest-even (numpy's astype(np.float32)); FLOAT32 passes through
 *     bit for bit. A FLOAT64 NaN becomes the quiet float NaN with the same sign and the top payload bits. Records are
 *     little-endian.
 *   - A frame whose layout has no intensity field (offset[3] < 0) is segmented exactly like an N x 3 frame (RNR skipped,
 *     S:379-382), even when other frames of the call carry intensity: its points get a NaN intensity, which no RNR test
 *     accepts, and the call runs with intensity on when any of its frames has it.
 *   - No byte outside [frames[f], frames[f] + n[f] * point_step) is read.
 *   - Checked before anything is allocated or launched (the message names the frame and the field); no stream's state
 *     changes on an error. PWPP_ERR_INVALID_ARG: a NULL streams / frames / n / layouts array, a NULL frame pointer with
 *     n > 0, n < 0, point_step < 1, an unknown datatype code, a field that does not fit inside point_step.
 *     PWPP_ERR_UNSUPPORTED: x / y / z not FLOAT32 or FLOAT64, point_step > PWPP_MAX_POINT_STEP.
 *   - After the call the unpacked points live in the ctx: every getter works as after the other entry points, and the xyz
 *     getters stay correct after the caller frees or reuses its record buffer.
 * pwpp_launch_count rises by one unpack launch per pipeline chunk that holds points (host) or per call (device). */
#define PWPP_FIELD_INT8 1    /* sensor_msgs/PointField datatype codes */
#define PWPP_FIELD_UINT8 2
#define PWPP_FIELD_INT16 3
#define PWPP_FIELD_UINT16 4
#define PWPP_FIELD_INT32 5
#define PWPP_FIELD_UINT32 6
#define PWPP_FIELD_FLOAT32 7
#define PWPP_FIELD_FLOAT64 8
#define PWPP_MAX_POINT_STEP 1024

typedef struct pwpp_point_layout {
  int32_t point_step;   /* bytes from one point to the next (PointCloud2::point_step), 1..PWPP_MAX_POINT_STEP */
  int32_t offset[4];    /* byte offsets of x, y, z, intensity inside a point; offset[3] < 0: no intensity field */
  int32_t datatype[4];  /* PWPP_FIELD_*; x, y, z must be FLOAT32 or FLOAT64, intensity any of the eight */
} pwpp_point_layout;

/* Host-resident records. Every frame's bytes travel as they are (no per-point host loop): a page-locked buffer by DMA
 * straight from it, a pageable one by one memcpy into page-locked staging and then DMA. The unpack runs on the upload stream
 * of the pipeline, so pwpp_call_times_us's host->device phase includes it. */
int pwpp_estimate_host_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames,
                               const int64_t* n, const pwpp_point_layout* layouts /* [nframes] */);
/* Device-resident records: unpacked on `cuda_stream` (NULL = the ctx's own stream) with the stream-ordering rules of
 * pwpp_estimate_device_xyz; the records must stay untouched until the call's work on that stream has run, and, when the
 * record results below are wanted, until they have been fetched (their gather reads the caller's buffers). */
int pwpp_estimate_device_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* d_frames,
                                 const int64_t* n, const pwpp_point_layout* layouts /* [nframes] */, void* cuda_stream);

/* Results of the last RECORDS call (pwpp_estimate_*_records) as records of each frame's own layout: every field the sensor
 * sent (intensity, ring, per-point time, padding) comes back byte for byte, so a ROS 2 node can publish its ground and
 * non-ground clouds with the input's fields. Frame f's region starts at byte h_offsets[f] (16-byte aligned; h_offsets has
 * nframes + 1 entries): num_ground(f) ground records, then num_nonground(f) non-ground records, in index-list order (record k
 * is input record k of the frame's lists, PWPP_ORDER_BIN or PWPP_ORDER_REFERENCE as the call ran); the bytes after them in
 * the region are unspecified.
 *   - The first of these four functions called after a call gathers the records of every frame in one kernel on the GPU
 *     (pwpp_launch_count rises by one; none for a call without points), on the call's stream; later calls of them reuse it.
 *     The host view adds one device->host copy into a page-locked buffer, and the per-frame getters copy from that. Calls
 *     that never ask for record results allocate and launch nothing for them.
 *   - Host blocking of pwpp_device_record_results: none once its buffers are warm, i.e. after a request of a call at least as
 *     large (in frames and record bytes). A request that first reserves or grows the output buffers or their page-locked
 *     offset table allocates device / page-locked memory, which the CUDA runtime may synchronize; and a request waits for the
 *     previous request's offset-table upload to have run (enqueued one call earlier, so in practice long done).
 *   - PWPP_ERR_INVALID_ARG before any call, for a frame outside the last call, and when the last call did not take records
 *     (the xyz getters serve those). Valid until the next estimate call. */
int pwpp_device_record_results(pwpp_ctx* ctx, const void** d_records, const int64_t** h_offsets);  /* enqueued on the call's stream; no host sync once warm */
int pwpp_host_record_results(pwpp_ctx* ctx, const void** h_records, const int64_t** h_offsets);    /* page-locked view, one D2H */
int pwpp_copy_ground_records(pwpp_ctx* ctx, int f, void* dst);       /* num_ground(f) * point_step bytes */
int pwpp_copy_nonground_records(pwpp_ctx* ctx, int f, void* dst);    /* num_nonground(f) * point_step bytes */

/* cudaDeviceSynchronize() on the ctx's device: what a binding calls before handing device memory produced on an unknown
 * stream to pwpp_estimate_device (and what makes its results visible to every stream afterwards). */
int pwpp_device_synchronize(pwpp_ctx* ctx);
int pwpp_synchronize(pwpp_ctx* ctx);

/* ---- results of the last estimate call, per frame f (position in the call) -------------- */

/* getGroundIndices / getNongroundIndices (H:159-160, S:18-26): int32 indices into the frame's
 * point array. Every input point appears in exactly one of the two lists (S:545-548).
 * Order: concentric-zone emission order of the reference (S:184-311) at bin granularity;
 * within one bin ascending point index (the reference's within-bin order is z-sorted with
 * implementation-defined ties, S:199). */
int64_t pwpp_num_ground(pwpp_ctx* ctx, int f);
int64_t pwpp_num_nonground(pwpp_ctx* ctx, int f);
int pwpp_copy_ground_indices(pwpp_ctx* ctx, int f, int32_t* dst);
int pwpp_copy_nonground_indices(pwpp_ctx* ctx, int f, int32_t* dst);
/* getGround / getNonground (H:157-158, S:8-16): row-major n x 3 float xyz of the listed points
 * (for RNR-rejected points the original z, S:393). */
int pwpp_copy_ground_xyz(pwpp_ctx* ctx, int f, float* dst);
int pwpp_copy_nonground_xyz(pwpp_ctx* ctx, int f, float* dst);
/* getCenters / getNormals (H:162-163, S:211-212): one row per bin that was plane-fitted
 * (>= num_min_pts points), in (zone, ring, sector) order; row-major k x 3 float. */
int pwpp_num_patches(pwpp_ctx* ctx, int f);
int pwpp_copy_centers(pwpp_ctx* ctx, int f, float* dst);
int pwpp_copy_normals(pwpp_ctx* ctx, int f, float* dst);
/* getHeight (H:154): the ADAPTIVE sensor height of STREAM f after its last frame (S:348). */
double pwpp_height(pwpp_ctx* ctx, int f);
/* getTimeTaken (H:155): microseconds of the last estimate call (whole call, all frames). */
double pwpp_time_us(pwpp_ctx* ctx);
/* Device-side split of that time for the last pwpp_estimate_host call, when the call ran as one chunk on one stream (calls of
 * a few frames — the reference's one-frame-per-call pattern): out = { host->device copy, kernels, device->host copy, all three }
 * in microseconds, from CUDA events on the call's stream. pwpp_time_us minus out[3] is host-side overhead. */
int pwpp_call_times_us(pwpp_ctx* ctx, float out[4]);

/* Device-side view of the index lists of the last call (zero-copy consumers, benchmark):
 * *d_indices -> int32 array laid out like the input (frame f's region starts at its point
 * offset); inside a region the ground list comes first, then the nonground list.
 * *d_num_ground -> int32[nframes]. Valid until the next estimate call. */
int pwpp_device_results(pwpp_ctx* ctx, const int32_t** d_indices, const int32_t** d_num_ground);

/* Order of the points INSIDE a bin's contribution to the index lists (the order of the bins, of the RNR / out-of-range
 * prefix and of the TGR-reverted patches is always the reference's, S:264-304):
 *   PWPP_ORDER_BIN        ascending point index (default of the C-ABI: what the fit kernels produce, no extra work);
 *   PWPP_ORDER_REFERENCE  the reference's order: ground part in ascending z; non-ground part = R-VPF removals by iteration,
 *                         each in ascending z, then the final rejects in ascending z (S:199, S:495-504, S:529-541); equal z
 *                         in ascending point index (= the reference with a stable per-bin sort). One extra kernel (a sort of
 *                         every fitted patch). The drop-in C++ class and pypatchworkpp select it by default.
 * Takes effect with the next estimate call. */
#define PWPP_ORDER_BIN 0
#define PWPP_ORDER_REFERENCE 1
int pwpp_set_output_order(pwpp_ctx* ctx, int order);

/* Host-side zero-copy view of the index lists of the last call (batch consumers: the per-frame getters above copy each
 * list once more, which for a 1024-frame batch is 0.5 GB of host memcpy): *h_indices -> the page-locked int32 buffer the
 * device lists were copied into, laid out like pwpp_device_results (frame f's region starts at point offset
 * *h_offsets[f]: ground list, then nonground list); *h_num_ground -> int32[nframes]. Fetches the lists from the device
 * if the call was a device-input call. Valid until the next estimate call. */
int pwpp_host_results(pwpp_ctx* ctx, const int32_t** h_indices, const int32_t** h_num_ground, const int64_t** h_offsets);

/* Placement helper for multi-GPU hosts: binds the CALLING THREAD (and with it the page-locked buffers it allocates
 * afterwards: first touch) to the CPUs of the NUMA node the device hangs off (sysfs numa_node / cpulist of its PCI
 * function). Returns the node (>= 0), or -1 if the topology could not be read (nothing changed). Call it before
 * pwpp_host_alloc / pwpp_create in a one-process-per-GPU launch. */
int pwpp_bind_host_to_device(int device);

/* ---- per-bin diagnostics for parity tests (not part of the reference surface) ------------ */

/* Per-bin record of the last call, frame f: bin ids in (zone,ring,sector) order. */
typedef struct pwpp_bin_result {
  double mean[3];      /* pc_mean_          (S:59-60) */
  double normal[3];    /* normal_, z >= 0   (S:66-68) */
  double sv[3];        /* singular_values_, descending (S:63) */
  double d;            /* d_                (S:74)    */
  int32_t n;           /* points binned into the patch (S:602-614) */
  int32_t n_ground;    /* |regionwise_ground_| (S:530)                 */
  int32_t verdict;     /* see PWPP_VERDICT_*                           */
  int32_t fitted;      /* 1 if n >= num_min_pts (S:191)                */
} pwpp_bin_result;

#define PWPP_VERDICT_SKIPPED 0        /* < num_min_pts: all nonground (S:191-195)  */
#define PWPP_VERDICT_NOT_UPRIGHT 1    /* S:262-265 */
#define PWPP_VERDICT_FAR_GROUND 2     /* S:266-269 */
#define PWPP_VERDICT_HEADING 3        /* S:270-273 */
#define PWPP_VERDICT_NEAR_GROUND 4    /* S:274-277 */
#define PWPP_VERDICT_TGR_REVERTED 5   /* S:444-450 */
#define PWPP_VERDICT_TGR_REJECTED 6   /* S:452-458, or enable_TGR == false (S:297-299) */

int pwpp_copy_bin_results(pwpp_ctx* ctx, int f, pwpp_bin_result* dst /* [nbins of frame f's set, <= pwpp_num_bins] */);
/* Polar bin id of every point of frame f as computed by the binning kernel:
 * 0..nbins-1, or nbins (= RNR hit, S:391-396) or nbins+1 (= outside (min_range,max_range], S:617-619). */
int pwpp_copy_bin_ids(pwpp_ctx* ctx, int f, uint16_t* dst /* [n_f] */);

/* ---- measurement hooks (not part of the reference surface) ---------------------------------- */

/* Page-locked host memory for callers that have no CUDA binding of their own. pwpp_estimate_host copies
 * straight from a caller buffer that is page-locked (allocated here, by cudaHostAlloc or registered with
 * cudaHostRegister) and row-major N x 4; any other buffer is first staged through the ctx's pinned buffer. */
void* pwpp_host_alloc(size_t bytes);
void pwpp_host_free(void* p);

#define PWPP_NUM_STAGES 11  /* bin_hist, bin_scan, scatter, fit_S, fit_L3, fit_L2, fit_L1, fit_M, fit_X, gle, emit */
/* With profiling on, CUDA events are recorded around every kernel of the following estimate calls;
 * pwpp_stage_times_ms() synchronizes and returns the device time of each stage of the LAST call. */
int pwpp_set_profiling(pwpp_ctx* ctx, int enabled);
int pwpp_stage_times_ms(pwpp_ctx* ctx, float* ms /* [PWPP_NUM_STAGES] */);
const char* pwpp_stage_name(int stage);
/* Number of kernels this ctx has launched since creation. */
int64_t pwpp_launch_count(const pwpp_ctx* ctx);

/* ---- temporal state (S:338-375), per STREAM f --------------------------------------------- */

int pwpp_get_state(pwpp_ctx* ctx, int f, pwpp_state* out);
/* Histories: ring r of update_elevation_ / update_flatness_ (H:174-175); dst holds n_* doubles. */
int pwpp_copy_history(pwpp_ctx* ctx, int f, int ring, int which /*0=elevation,1=flatness*/, double* dst);
/* Checkpoint / migration of one stream (SURVEY.md 8f-4): the COMPLETE temporal state the reference object carries from
 * frame to frame — adaptive sensor height and thresholds (S:347-350, S:368), both history arrays (H:174-175) and the
 * plane members left by the last estimate_plane call (S:49 keeps them when a patch's seed set is empty) — as one
 * opaque blob. A blob exported from stream f of one ctx can be imported into any stream of any ctx created with the
 * same parameters (another GPU, another process, a later run): the next frame then gives bit-identical results.
 * pwpp_export_state synchronizes with the last estimate call; pwpp_import_state takes effect before the next one. */
size_t pwpp_state_blob_size(const pwpp_ctx* ctx);           /* the largest over the sets: fits any stream's blob */
size_t pwpp_stream_state_blob_size(const pwpp_ctx* ctx, int s); /* the blob of stream s (its set's hist_cap); 0 for a bad s */
int pwpp_export_state(pwpp_ctx* ctx, int f, void* blob /* [pwpp_state_blob_size] */);
int pwpp_import_state(pwpp_ctx* ctx, int f, const void* blob, size_t bytes);
/* Re-initialises stream f / all streams to the constructor state (a fresh PatchWorkpp instance).
 * Stream-ordered: enqueued behind the last estimate call, no host synchronization. */
int pwpp_reset_stream(pwpp_ctx* ctx, int f);
int pwpp_reset_all(pwpp_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* PWPP_H_ */
