// kinfu_snapshot.cu -- snapshots of the frame loop's state: df_kinfu_save / df_kinfu_load / df_kinfu_snapshot_params /
// df_kinfu_snapshot_color_camera / df_kinfu_snapshot_lenses.  The format is spelled out in dfusion.h; the volumes travel brick-packed (snapshot.cu).
#include "kinfu_object.cuh"
#include "lens.cuh"
#include <cstdio>

using namespace dfb::kinfu;

namespace {

constexpr char SNAP_MAGIC[8] = {'D', 'F', 'U', 'S', 'N', 'A', 'P', '\0'};
// version 1; version 2 (objects with DF_KINFU_COLOR) appends the colour sections; version 3 (a colour camera set) then its calibration;
// version 4 (a lens set) any of those, then the lens section; version 5 (DF_KINFU_RELOCALISE) any of those, then the relocaliser section
uint32_t snap_version(const df_kinfu_params &p, bool camera, bool lenses)
{
    return lenses ? 4u : (p.flags & DF_KINFU_COLOR) ? (camera ? 3u : 2u) : 1u;
}
static_assert(sizeof(df_color_camera) == 72, "the version-3 camera record is a byte copy of df_color_camera");
static_assert(sizeof(df_lens) == 36, "the version-4 lens records are byte copies of df_lens");
constexpr size_t LENS_SECTION = 2 * (1 + sizeof(df_lens));   // u8 present + record, for the depth lens, then the colour lens

struct SnapHeader {
    char magic[8];
    uint32_t version, header_bytes;
    uint64_t total_bytes, checksum;        // checksum of bytes [header_bytes, total_bytes)
};
struct SnapCounters {
    int32_t frame_counter, resets, last_ok, M, cloud_count, n_poses;
    int64_t solve_overflows;
    uint64_t payload_bytes;
};
// the head of the version-5 relocaliser section; then count x n_ferns code bytes, count x 12 pose floats, and the u64 section length
struct RelocSection {
    uint32_t base_version;                 // the version (1-4) the rest of the snapshot has
    uint8_t lost, pad[3];
    int64_t lost_frames, relocalisations;
    uint64_t seed;
    int32_t count, n_ferns;
};
static_assert(sizeof(SnapHeader) == 32 && sizeof(SnapCounters) == 40 && sizeof(RelocSection) == 40, "snapshot sections are packed");
size_t reloc_section_bytes(int count) { return sizeof(RelocSection) + (size_t)count * (DF_RELOC_FERNS + 48) + 8; }

// sum over the little-endian u64 words w_i of the (zero-padded) body of splitmix64(w_i ^ i * golden), plus the length
uint64_t snap_checksum(const unsigned char *p, size_t n)
{
    uint64_t acc = 0;
    const size_t nw = (n + 7) / 8;
    for (size_t i = 0; i < nw; ++i) {
        uint64_t w = 0;
        memcpy(&w, p + 8 * i, n - 8 * i < 8 ? n - 8 * i : 8);
        uint64_t z = w ^ (i * 0x9e3779b97f4a7c15ull);
        z += 0x9e3779b97f4a7c15ull;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        acc += z ^ (z >> 31);
    }
    return acc + (uint64_t)n;
}

// byte offsets of the sections, all derived from the params and the counters
struct SnapLayout {
    df_kinfu_params p; df_f2_params f2; SnapCounters c;
    int levels; size_t activity_bytes, nbricks;
    size_t poses, nodes, activity, pyr, pyr_bytes, cloud, cloud_nrm, classes, payload, total;
    // version 2: u64 color_payload_bytes at color_len, then the colour volume's class bytes and payload, then cloud_count RGBA words
    uint64_t color_payload_bytes = 0;
    size_t color_len = 0, color_classes = 0, color_payload = 0, cloud_rgba = 0;
    // version 3: the df_color_camera record at `camera`
    bool has_camera = false;
    size_t camera = 0;
    // version 4: the lens section at `lenses`
    bool has_lenses = false;
    size_t lenses = 0;
    // version 5: the relocaliser section at `reloc`
    bool has_reloc = false;
    RelocSection r = {};
    size_t reloc = 0;
};

df_volume geometry_of(const df_kinfu_params &p)
{
    df_volume v = {};
    for (int i = 0; i < 3; ++i) v.dims[i] = p.volume_dims[i];
    return v;
}

// levels x (points or depth + normals), dense rows, level l = (cols >> l) x (rows >> l)
size_t pyramid_bytes(const df_kinfu_params &p, int levels)
{
    size_t n = 0;
    const size_t first = (p.flags & DF_KINFU_USE_DEPTH) ? 2 : 16;
    int cols = p.cols, rows = p.rows;
    for (int l = 0; l < levels; ++l, cols /= 2, rows /= 2) n += (size_t)cols * rows * (first + 16);
    return n;
}

void layout_sections(SnapLayout &L)
{
    const SnapCounters &c = L.c;
    L.levels = used_levels(L.p);
    const df_volume v = geometry_of(L.p);
    L.activity_bytes = df_volume_activity_bytes(v);
    L.nbricks = df_volume_brick_count(v);
    size_t o = sizeof(SnapHeader) + sizeof(df_kinfu_params) + sizeof(df_f2_params) + sizeof(SnapCounters);
    L.poses = o; o += (size_t)c.n_poses * 48;
    L.nodes = o; o += (size_t)c.M * DF_NODE_STRIDE * 4;
    L.activity = o; o += L.activity_bytes;
    L.pyr = o; L.pyr_bytes = pyramid_bytes(L.p, L.levels); o += L.pyr_bytes;
    L.cloud = o; o += (size_t)c.cloud_count * 16;
    L.cloud_nrm = o; o += (size_t)c.cloud_count * 16;
    L.classes = o; o += L.nbricks;
    L.payload = o; o += c.payload_bytes;
    if (L.p.flags & DF_KINFU_COLOR) {
        L.color_len = o; o += 8;
        L.color_classes = o; o += L.nbricks;
        L.color_payload = o; o += L.color_payload_bytes;
        L.cloud_rgba = o; o += (size_t)c.cloud_count * 4;
    }
    if (L.has_camera) { L.camera = o; o += sizeof(df_color_camera); }
    if (L.has_lenses) { L.lenses = o; o += LENS_SECTION; }
    if (L.has_reloc) { L.reloc = o; o += reloc_section_bytes(L.r.count); }
    L.total = o;
}

int reject(const char *why)
{
    fprintf(stderr, "df_kinfu snapshot rejected: %s\n", why);
    return (int)cudaErrorInvalidValue;
}

// every check that needs only the bytes: header, checksum, counters, section lengths
int parse_snapshot(const void *buf, size_t bytes, SnapLayout &L)
{
    const unsigned char *b = (const unsigned char *)buf;
    const size_t fixed = sizeof(SnapHeader) + sizeof(df_kinfu_params) + sizeof(df_f2_params) + sizeof(SnapCounters);
    if (!buf || bytes < sizeof(SnapHeader)) return reject("shorter than the header");
    SnapHeader h;
    memcpy(&h, b, sizeof h);
    if (memcmp(h.magic, SNAP_MAGIC, 8) != 0) return reject("not a snapshot (magic)");
    if (h.version < 1 || h.version > 5) return reject("unsupported format version");
    if (h.header_bytes != sizeof(SnapHeader)) return reject("header length");
    if (h.total_bytes != bytes) return reject("length differs from the header's (truncated or padded)");
    if (bytes < fixed) return reject("shorter than its fixed sections");
    if (snap_checksum(b + sizeof h, bytes - sizeof h) != h.checksum) return reject("checksum mismatch");
    size_t o = sizeof h;
    memcpy(&L.p, b + o, sizeof L.p); o += sizeof L.p;
    memcpy(&L.f2, b + o, sizeof L.f2); o += sizeof L.f2;
    memcpy(&L.c, b + o, sizeof L.c);
    const SnapCounters &c = L.c;
    const df_kinfu_params &p = L.p;
    // version 5: the relocaliser section ends the snapshot and its last 8 bytes give its length; the rest is a snapshot of its base version
    uint32_t version = h.version;
    L.has_reloc = version == 5;
    if (L.has_reloc) {
        uint64_t len = 0;
        if (bytes < fixed + reloc_section_bytes(0)) return reject("relocaliser section lengths (truncated)");
        memcpy(&len, b + bytes - 8, 8);
        if (len < reloc_section_bytes(0) || len > bytes - fixed) return reject("relocaliser section lengths");
        memcpy(&L.r, b + bytes - len, sizeof L.r);
        const RelocSection &r = L.r;
        if (r.base_version < 1 || r.base_version > 4) return reject("relocaliser section: base version");
        if (r.count < 0 || r.count > DF_RELOC_KEYFRAMES) return reject("relocaliser section: more keyframes than the database holds");
        if (r.n_ferns != DF_RELOC_FERNS || r.seed != DF_RELOC_SEED) return reject("relocaliser section: fern table differs from this library's");
        if (r.lost > 1 || r.pad[0] || r.pad[1] || r.pad[2] || r.lost_frames < 0 || r.relocalisations < 0) return reject("relocaliser section: counters");
        if (len != reloc_section_bytes(r.count)) return reject("relocaliser section lengths");
        version = r.base_version;
        bytes -= len;                                                  // the checks below see the base snapshot
    }
    if (L.has_reloc != ((p.flags & DF_KINFU_RELOCALISE) != 0)) return reject("relocaliser section does not match the DF_KINFU_RELOCALISE flag of its parameters");
    if (p.volume_dims[0] <= 0 || p.volume_dims[0] % 32 || p.volume_dims[1] <= 0 || p.volume_dims[2] <= 0 || p.cols <= 0 || p.rows <= 0 ||
        p.cloud_capacity < 0)
        return reject("parameters");
    if ((double)p.volume_dims[0] * p.volume_dims[1] * p.volume_dims[2] >= 2147483648.0 || (double)p.cols * p.rows >= 2147483648.0)
        return reject("parameters");
    if (c.frame_counter < 0 || c.resets < 0 || c.M < 0 || c.cloud_count < 0 || c.n_poses < 1 || c.solve_overflows < 0) return reject("counters");
    if (c.payload_bytes % 4 || c.payload_bytes > 4 * (size_t)df_volume_brick_count(geometry_of(p)) * DF_BRICK * DF_BRICK * DF_BRICK ||
        (double)c.n_poses * 48 > (double)bytes || c.cloud_count > p.cloud_capacity)
        return reject("section lengths");
    L.has_camera = version == 3;
    L.has_lenses = version == 4;
    if (!L.has_lenses && version != snap_version(p, L.has_camera, false)) return reject("format version does not match the colour flag of its parameters");
    L.color_payload_bytes = 0;
    layout_sections(L);
    if (p.flags & DF_KINFU_COLOR) {
        if (L.color_len + 8 > bytes) return reject("colour section lengths");
        memcpy(&L.color_payload_bytes, b + L.color_len, 8);
        if (L.color_payload_bytes > bytes) return reject("colour section lengths");
        layout_sections(L);
        // version 4 of a colour object: the camera record is there when the length says so
        const size_t reloc_bytes = L.has_reloc ? reloc_section_bytes(L.r.count) : 0;
        if (L.has_lenses && L.total - reloc_bytes + sizeof(df_color_camera) == bytes) { L.has_camera = true; layout_sections(L); }
    }
    if (L.total != bytes + (L.has_reloc ? reloc_section_bytes(L.r.count) : 0))
        return reject(L.color_len ? "section lengths (colour sections included)" : "section lengths");
    if (L.has_lenses) {
        const unsigned char *ls = b + L.lenses;
        bool any = false;
        for (int i = 0; i < 2; ++i, ls += 1 + sizeof(df_lens)) {
            df_lens lens;
            memcpy(&lens, ls + 1, sizeof lens);
            if (ls[0] > 1) return reject("a lens presence byte is not 0 or 1");
            if (ls[0] && (df_lens_check(lens) != 0 || dfb::lens_is_zero(lens))) return reject("lens record");
            static const unsigned char zero[sizeof(df_lens)] = {};
            if (!ls[0] && memcmp(ls + 1, zero, sizeof zero) != 0) return reject("a lens record that is not present is not zero");
            any = any || ls[0];
        }
        if (!any) return reject("version 4 without a lens");
        if (b[L.lenses + 1 + sizeof(df_lens)] && !L.has_camera) return reject("a colour lens without a colour camera record");
    }
    if (L.has_camera) {
        df_color_camera cam;
        memcpy(&cam, b + L.camera, sizeof cam);
        if (df_color_map_dims(p.intr, cam, nullptr, nullptr, nullptr) != 0) return reject("colour camera record");
    }
    if (p.flags & DF_KINFU_COLOR) {
        // the brick rule of df_volume_unpack, checked here so that a load can refuse before it writes either volume
        uint64_t words = 0;
        for (size_t i = 0; i < L.nbricks; ++i) {
            const unsigned char cls = b[L.color_classes + i];
            if (cls > 2) return reject("a colour brick class byte is not 0, 1 or 2");
            words += cls == 2 ? (uint64_t)DF_BRICK * DF_BRICK * DF_BRICK : cls;
        }
        if (4 * words != L.color_payload_bytes) return reject("colour payload length differs from what its brick classes imply");
    }
    return 0;
}

// the sections that are object buffers byte for byte, in snapshot order: fn(device pointer, offset in the snapshot, length)
template <class F> int for_each_buffer_section(KinFu &k, const SnapLayout &L, F &&fn)
{
    CK(fn(k.nodes.p, L.nodes, (size_t)L.c.M * DF_NODE_STRIDE * 4));
    CK(fn(k.activity.p, L.activity, L.activity_bytes));
    size_t o = L.pyr;
    for (int l = 0; l < L.levels; ++l) {
        const Img &first = (k.p.flags & DF_KINFU_USE_DEPTH) ? k.prev_depth[l] : k.prev_pts[l];
        const Img *ims[2] = {&first, &k.prev_nrm[l]};
        for (const Img *im : ims) {
            CK(fn(im->ptr, o, im->pitch * im->rows));
            o += im->pitch * im->rows;
        }
    }
    CK(fn(k.cloud.p, L.cloud, (size_t)L.c.cloud_count * 16));
    CK(fn(k.cloud_nrm.p, L.cloud_nrm, (size_t)L.c.cloud_count * 16));
    return 0;
}

// a volume packed for the snapshot: df_volume_pack_count (class bytes and payload length, one host synchronisation), then emit()
struct PackedVolume {
    DevMem<void> ws; DevMem<unsigned char> classes; DevMem<unsigned long long> len; DevMem<uint32_t> payload;
    unsigned long long bytes = 0;

    int count(const df_volume &v, cudaStream_t s)
    {
        CK(ws.alloc(df_volume_pack_workspace_bytes(v)));
        CK(classes.alloc(df_volume_brick_count(v)));
        CK(len.alloc(8));
        CK(df_volume_pack_count(v, ws, classes, len, s));
        CK(cudaMemcpyAsync(&bytes, len, 8, cudaMemcpyDeviceToHost, s));
        return (int)cudaStreamSynchronize(s);
    }
    // df_volume_pack_emit, then the class bytes and the payload into the snapshot at `classes_at` and `payload_at`
    int emit(const df_volume &v, unsigned char *classes_at, unsigned char *payload_at, cudaStream_t s)
    {
        CK(payload.alloc(bytes));
        CK(df_volume_pack_emit(v, ws, classes, payload, bytes, s));
        CK(cudaMemcpyAsync(classes_at, classes, df_volume_brick_count(v), cudaMemcpyDeviceToHost, s));
        return (int)cudaMemcpyAsync(payload_at, payload, bytes, cudaMemcpyDeviceToHost, s);
    }
};

// the snapshot's class bytes and payload of a packed volume into `v` (df_volume_unpack), or a rejection from its status
int unpack_volume(const df_volume &v, const unsigned char *classes_at, const unsigned char *payload_at, uint64_t bytes, cudaStream_t s)
{
    const size_t nbricks = df_volume_brick_count(v);
    DevMem<void> ws; DevMem<unsigned char> classes; DevMem<uint32_t> payload; DevMem<int> st;
    CK(ws.alloc(df_volume_pack_workspace_bytes(v)));
    CK(classes.alloc(nbricks));
    CK(payload.alloc(bytes));
    CK(st.alloc(sizeof(int)));
    CK(cudaMemcpyAsync(classes, classes_at, nbricks, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(payload, payload_at, bytes, cudaMemcpyHostToDevice, s));
    CK(df_volume_unpack(v, classes, payload, bytes, ws, st, s));
    int status = 0;
    CK(cudaMemcpyAsync(&status, st, sizeof status, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));                                      // the staging buffers are released on return
    if (status == DF_UNPACK_BAD_CLASS) return reject("a brick class byte is not 0, 1 or 2");
    return status ? reject("payload length differs from what the brick classes imply") : 0;
}

}  // namespace

extern "C" int df_kinfu_snapshot_params(const void *buf, size_t bytes, df_kinfu_params *params)
{
    if (!params) return (int)cudaErrorInvalidValue;
    SnapLayout L;
    if (int st = parse_snapshot(buf, bytes, L)) return st;
    *params = L.p;
    return 0;
}

extern "C" int df_kinfu_snapshot_color_camera(const void *buf, size_t bytes, df_color_camera *cam, int *present)
{
    if (!present) return (int)cudaErrorInvalidValue;
    SnapLayout L;
    if (int st = parse_snapshot(buf, bytes, L)) return st;
    *present = L.has_camera;
    if (cam) {
        if (L.has_camera) memcpy(cam, (const unsigned char *)buf + L.camera, sizeof *cam);
        else memset(cam, 0, sizeof *cam);
    }
    return 0;
}

extern "C" int df_kinfu_snapshot_lenses(const void *buf, size_t bytes, df_lens *depth, int *depth_present, df_lens *color, int *color_present)
{
    if (!depth_present || !color_present) return (int)cudaErrorInvalidValue;
    SnapLayout L;
    if (int st = parse_snapshot(buf, bytes, L)) return st;
    const unsigned char *ls = (const unsigned char *)buf + L.lenses;
    int *present[2] = {depth_present, color_present};
    df_lens *out[2] = {depth, color};
    for (int i = 0; i < 2; ++i, ls += 1 + sizeof(df_lens)) {
        *present[i] = L.has_lenses ? ls[0] : 0;
        if (out[i]) {
            if (*present[i]) memcpy(out[i], ls + 1, sizeof(df_lens));
            else memset(out[i], 0, sizeof(df_lens));
        }
    }
    return 0;
}

extern "C" int df_kinfu_save(void *h, void *dst_host, size_t capacity, size_t *bytes_out)
{
    KinFu *k = (KinFu *)h;
    if (!k) return (int)cudaErrorInvalidValue;
    cudaSetDevice(k->device);
    cudaStream_t s = k->stream;
    sync_extract(*k);                                                  // the cloud of the last frame is complete
    CK(cudaStreamSynchronize(s));
    note_solve_overflow(*k);
    SnapLayout L;
    L.p = k->p; L.f2 = k->f2;
    int count = 0;
    CK(cudaMemcpy(&count, k->cloud_count, sizeof count, cudaMemcpyDeviceToHost));
    L.c = SnapCounters{k->frame_counter, k->resets, k->last_ok, k->M, count, (int32_t)(k->poses.size() / 12), k->solve_overflows, 0};
    PackedVolume vol, col;                                             // the TSDF volume and, under DF_KINFU_COLOR, the colour volume
    CK(vol.count(vol_of(*k), s));
    if (color_on(*k)) CK(col.count(color_vol_of(*k), s));
    L.c.payload_bytes = vol.bytes;
    L.color_payload_bytes = col.bytes;
    L.has_camera = k->has_cam;
    L.has_lenses = k->has_depth_lens || k->has_color_lens;
    L.has_reloc = reloc_on(*k);
    if (L.has_reloc) {
        int kf = 0;
        CK(cudaMemcpy(&kf, k->kf_count, sizeof kf, cudaMemcpyDeviceToHost));
        L.r = RelocSection{snap_version(L.p, L.has_camera, L.has_lenses), (uint8_t)k->lost, {0, 0, 0}, k->lost_frames, k->relocalisations,
                           DF_RELOC_SEED, kf, DF_RELOC_FERNS};
    }
    layout_sections(L);
    if (bytes_out) *bytes_out = L.total;
    if (!dst_host) return 0;
    if (capacity < L.total) return (int)cudaErrorInvalidValue;
    unsigned char *b = (unsigned char *)dst_host;
    size_t o = sizeof(SnapHeader);
    memcpy(b + o, &L.p, sizeof L.p); o += sizeof L.p;
    memcpy(b + o, &L.f2, sizeof L.f2); o += sizeof L.f2;
    memcpy(b + o, &L.c, sizeof L.c);
    memcpy(b + L.poses, k->poses.data(), (size_t)L.c.n_poses * 48);
    CK(vol.emit(vol_of(*k), b + L.classes, b + L.payload, s));
    CK(for_each_buffer_section(*k, L, [&](void *dev, size_t off, size_t n) { return cudaMemcpyAsync(b + off, dev, n, cudaMemcpyDeviceToHost, s); }));
    if (color_on(*k)) {
        const uint64_t len = col.bytes;
        memcpy(b + L.color_len, &len, 8);
        CK(col.emit(color_vol_of(*k), b + L.color_classes, b + L.color_payload, s));
        CK(cudaMemcpyAsync(b + L.cloud_rgba, k->cloud_rgba, (size_t)L.c.cloud_count * 4, cudaMemcpyDeviceToHost, s));
    }
    if (L.has_camera) memcpy(b + L.camera, &k->cam, sizeof k->cam);
    if (L.has_lenses) {
        unsigned char *ls = b + L.lenses;
        ls[0] = k->has_depth_lens; memcpy(ls + 1, &k->depth_lens, sizeof(df_lens));
        ls += 1 + sizeof(df_lens);
        ls[0] = k->has_color_lens; memcpy(ls + 1, &k->color_lens, sizeof(df_lens));
    }
    if (L.has_reloc) {
        unsigned char *r = b + L.reloc;
        memcpy(r, &L.r, sizeof L.r);
        r += sizeof L.r;
        CK(cudaMemcpyAsync(r, k->kf_codes, (size_t)L.r.count * DF_RELOC_FERNS, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(r + (size_t)L.r.count * DF_RELOC_FERNS, k->kf_poses, (size_t)L.r.count * 48, cudaMemcpyDeviceToHost, s));
        const uint64_t len = reloc_section_bytes(L.r.count);
        memcpy(b + L.total - 8, &len, 8);
    }
    CK(cudaStreamSynchronize(s));
    SnapHeader hd;
    memcpy(hd.magic, SNAP_MAGIC, 8);
    hd.version = L.has_reloc ? 5u : snap_version(L.p, L.has_camera, L.has_lenses); hd.header_bytes = sizeof hd; hd.total_bytes = L.total;
    hd.checksum = snap_checksum(b + sizeof hd, L.total - sizeof hd);
    memcpy(b, &hd, sizeof hd);
    return 0;
}

extern "C" int df_kinfu_load(void *h, const void *src_host, size_t bytes)
{
    KinFu *k = (KinFu *)h;
    if (!k) return (int)cudaErrorInvalidValue;
    SnapLayout L;
    if (int st = parse_snapshot(src_host, bytes, L)) return st;
    if (memcmp(&L.p, &k->p, sizeof L.p) != 0) return reject("parameters differ from the object's");
    if (L.has_camera != k->has_cam || (L.has_camera && memcmp((const unsigned char *)src_host + L.camera, &k->cam, sizeof k->cam) != 0))
        return reject("colour camera differs from the object's (df_kinfu_set_color_camera before loading)");
    {
        // the object's lenses as the lens section would record them (no section: none set)
        unsigned char mine[LENS_SECTION] = {}, theirs[LENS_SECTION] = {};
        mine[0] = k->has_depth_lens; memcpy(mine + 1, &k->depth_lens, sizeof(df_lens));
        mine[1 + sizeof(df_lens)] = k->has_color_lens; memcpy(mine + 2 + sizeof(df_lens), &k->color_lens, sizeof(df_lens));
        if (L.has_lenses) memcpy(theirs, (const unsigned char *)src_host + L.lenses, LENS_SECTION);
        if (memcmp(mine, theirs, LENS_SECTION) != 0)
            return reject("lenses differ from the object's (df_kinfu_set_depth_lens / _set_color_lens before loading)");
    }
    if (L.c.M > k->max_nodes_cap) return reject("more nodes than the object can hold");
    cudaSetDevice(k->device);
    cudaStream_t s = k->stream;
    sync_extract(*k);                                                  // nothing may still read or write the buffers below
    k->extract_pending = false;
    CK(cudaStreamSynchronize(s));
    note_solve_overflow(*k);
    const unsigned char *b = (const unsigned char *)src_host;
    CK(unpack_volume(vol_of(*k), b + L.classes, b + L.payload, L.c.payload_bytes, s));
    // the volume is in place; nothing below can fail on the snapshot's contents (parse_snapshot has checked the colour bricks)
    if (color_on(*k)) {
        CK(unpack_volume(color_vol_of(*k), b + L.color_classes, b + L.color_payload, L.color_payload_bytes, s));
        CK(cudaMemcpyAsync(k->cloud_rgba, b + L.cloud_rgba, (size_t)L.c.cloud_count * 4, cudaMemcpyHostToDevice, s));
    }
    CK(for_each_buffer_section(*k, L, [&](void *dev, size_t off, size_t n) { return cudaMemcpyAsync(dev, b + off, n, cudaMemcpyHostToDevice, s); }));
    CK(cudaMemcpyAsync(k->cloud_count, &L.c.cloud_count, sizeof(int), cudaMemcpyHostToDevice, s));
    if (L.has_reloc) {                                                 // the parameters match, so the object has the flag and its buffers
        const unsigned char *r = b + L.reloc + sizeof(RelocSection);
        CK(cudaMemcpyAsync(k->kf_codes, r, (size_t)L.r.count * DF_RELOC_FERNS, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(k->kf_poses, r + (size_t)L.r.count * DF_RELOC_FERNS, (size_t)L.r.count * 48, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(k->kf_count, &L.r.count, sizeof(int), cudaMemcpyHostToDevice, s));
    }
    if (L.c.M > 0) CK(df_build_node_grid(k->nodes, L.c.M, k->node_grid, s));
    CK(cudaStreamSynchronize(s));
    k->f2 = L.f2;
    k->frame_counter = L.c.frame_counter; k->resets = L.c.resets; k->last_ok = L.c.last_ok; k->M = L.c.M;
    k->solve_overflows = L.c.solve_overflows;
    if (L.has_reloc) { k->lost = L.r.lost != 0; k->lost_frames = L.r.lost_frames; k->relocalisations = L.r.relocalisations; }
    k->last_cloud = L.c.cloud_count;
    k->poses.resize((size_t)L.c.n_poses * 12);
    memcpy(k->poses.data(), b + L.poses, (size_t)L.c.n_poses * 48);
    k->extract_deferred = false; k->extract_pending = false;
    k->lm_valid = false;                                               // DF_KINFU_LIVE_MODEL: the next frame builds it from the loaded state
    return 0;
}
