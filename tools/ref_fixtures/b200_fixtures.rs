//! Reference-side fixture generator for cosdata-b200 (tools/ref_fixtures/README.md).
//!
//! Drop this file into the cosdata crate as `tests/b200_fixtures.rs` and run
//!
//!     CDB_FIXTURE_DIR=/path/to/cosdata-b200/tests/golden/ref \
//!         cargo test --release --test b200_fixtures -- --nocapture
//!
//! It calls the crate's OWN hot-path functions (nothing is restated here except the synthetic
//! input generator, which must produce the same f32 values as include/cosdata_b200.h) and writes
//!   hotpath_ref_v1.cdbf   quantize / dot_product_* / DistanceMetric::calculate / PerformantFixedSet results
//!   prop.data             write_prop_value_to_file records (file_persist.rs:70-90)
//!   itoe.dim, itoe.0.data TreeMap<InternalId, RawVectorEmbedding> (collection.rs:149-164)
//!   tf_idf_index/         index-tree.dim and <version>.idat of a TFIDFIndexRoot (tf_idf_index.rs), 3 versions
//! for the same inputs as tests/golden/make_golden.py.  tests/test_golden.py and the reader tests of
//! cosdata-b200 pick the files up when present and compare them with the oracle, the committed
//! golden vectors and the CUDA path.
//!
//! Record format of the .cdbf container (little endian):
//!   u32 name_len, name bytes, u32 dtype (0 u8, 1 i8, 2 u32, 3 f32), u32 ndim, u64 dims[ndim], payload.

use std::fs::{File, OpenOptions};
use std::io::Write;
use std::path::PathBuf;
use std::sync::Arc;

use cosdata::distance::{DistanceError, DistanceFunction};
use cosdata::models::buffered_io::{BufferManager, BufferManagerFactory};
use cosdata::models::collection::RawVectorEmbedding;
use cosdata::models::dot_product::{
    dot_product_binary, dot_product_f16, dot_product_f32, dot_product_octal, dot_product_quaternary,
    dot_product_u8,
};
use cosdata::models::file_persist::{write_prop_metadata_to_file, write_prop_value_to_file};
use cosdata::models::fixedset::PerformantFixedSet;
use cosdata::models::tf_idf_index::TFIDFIndexRoot;
use cosdata::models::tree_map::TreeMap;
use cosdata::models::types::{DistanceMetric, InternalId, Metadata, VectorData, VectorId};
use cosdata::models::versioning::VersionNumber;
use cosdata::quantization::scalar::ScalarQuantization;
use cosdata::quantization::{Quantization, StorageType};
use cosdata::storage::Storage;

// ---------------------------------------------------------------- synthetic inputs
// include/cosdata_b200.h: element idx of stream `seed`
fn synth_value(seed: u64, idx: u64) -> f32 {
    let mut z = seed.wrapping_add(idx.wrapping_mul(0x9E3779B97F4A7C15));
    z = (z ^ (z >> 30)).wrapping_mul(0xBF58476D1CE4E5B9);
    z = (z ^ (z >> 27)).wrapping_mul(0x94D049BB133111EB);
    z ^= z >> 31;
    let m = ((z >> 40) as i32) - (1 << 23);
    (m as f32) * (1.0f32 / 8388608.0f32)
}

fn synth_matrix(seed: u64, n: usize, dim: usize) -> Vec<Vec<f32>> {
    (0..n)
        .map(|r| (0..dim).map(|c| synth_value(seed, (r * dim + c) as u64)).collect())
        .collect()
}

fn edge_values() -> Vec<f32> {
    vec![
        -1.0, 1.0, 0.0, -0.0, 1.5, -1.5, 0.99999994, -0.99999994, 1e-40, -1e-40, 0.5, -0.5, 0.25, 0.75,
        5.9604645e-8,  // 2^-24
        -5.9604645e-8,
    ]
}

// tests/golden/make_golden.py::corpus_for
fn corpus_for(dim: usize) -> (Vec<Vec<f32>>, Vec<Vec<f32>>) {
    let n = if dim <= 128 { 16 } else { 8 };
    let edge = edge_values();
    let mut m = synth_matrix(0x601D + dim as u64, n, dim);
    for c in 0..dim {
        m[0][c] = 0.0;
        m[1][c] = edge[c % edge.len()];
    }
    m[3] = m[2].clone();
    m[4] = m[2].iter().map(|x| -x).collect();
    let mut q = synth_matrix(0x9E57 + dim as u64, 3, dim);
    q[1] = m[2].clone();
    for c in 0..dim.min(edge.len()) {
        q[2][c] = edge[c];
    }
    (m, q)
}

// ---------------------------------------------------------------- container
struct Out {
    f: File,
}
impl Out {
    fn rec(&mut self, name: &str, dtype: u32, dims: &[u64], payload: &[u8]) {
        self.f.write_all(&(name.len() as u32).to_le_bytes()).unwrap();
        self.f.write_all(name.as_bytes()).unwrap();
        self.f.write_all(&dtype.to_le_bytes()).unwrap();
        self.f.write_all(&(dims.len() as u32).to_le_bytes()).unwrap();
        for d in dims {
            self.f.write_all(&d.to_le_bytes()).unwrap();
        }
        self.f.write_all(payload).unwrap();
    }
    fn u8s(&mut self, name: &str, dims: &[u64], v: &[u8]) {
        self.rec(name, 0, dims, v);
    }
    fn i8s(&mut self, name: &str, dims: &[u64], v: &[i8]) {
        let b: Vec<u8> = v.iter().map(|x| *x as u8).collect();
        self.rec(name, 1, dims, &b);
    }
    fn u32s(&mut self, name: &str, dims: &[u64], v: &[u32]) {
        let b: Vec<u8> = v.iter().flat_map(|x| x.to_le_bytes()).collect();
        self.rec(name, 2, dims, &b);
    }
    fn f32s(&mut self, name: &str, dims: &[u64], v: &[f32]) {
        let b: Vec<u8> = v.iter().flat_map(|x| x.to_le_bytes()).collect();
        self.rec(name, 3, dims, &b);
    }
}

// tight code layout of cosdata_b200.h::cdb_code_bytes: u8 D | sub r planes of ceil(D/8) bytes, plane 0 first | f16 2D | f32 4D
fn code_bytes(s: &Storage) -> Vec<u8> {
    match s {
        Storage::UnsignedByte { quant_vec, .. } => quant_vec.clone(),
        Storage::SubByte { quant_vec, .. } => quant_vec.iter().flat_map(|p| p.iter().copied()).collect(),
        Storage::HalfPrecisionFP { quant_vec, .. } => quant_vec.iter().flat_map(|h| h.to_bits().to_le_bytes()).collect(),
        Storage::FullPrecisionFP { vec, .. } => vec.iter().flat_map(|x| x.to_le_bytes()).collect(),
    }
}
fn mag_of(s: &Storage) -> f32 {
    match s {
        Storage::UnsignedByte { mag, .. }
        | Storage::SubByte { mag, .. }
        | Storage::HalfPrecisionFP { mag, .. }
        | Storage::FullPrecisionFP { mag, .. } => *mag,
    }
}
fn storage_type(st: u32) -> StorageType {
    match st {
        0 => StorageType::UnsignedByte,
        1 | 2 | 3 => StorageType::SubByte(st as u8),
        4 => StorageType::HalfPrecisionFP,
        _ => StorageType::FullPrecisionFP,
    }
}
fn metric_of(m: u32) -> DistanceMetric {
    match m {
        0 => DistanceMetric::Cosine,
        1 => DistanceMetric::Euclidean,
        2 => DistanceMetric::Hamming,
        _ => DistanceMetric::DotProduct,
    }
}

// (status, value): 0 Ok, 1 StorageMismatch, 2 CalculationError, 6 the reference panicked (unimplemented!())
fn calc(metric: u32, x: &Storage, y: &Storage) -> (i8, f32) {
    let r = std::panic::catch_unwind(|| {
        let xd = VectorData::without_metadata(None, x);
        let yd = VectorData::without_metadata(None, y);
        metric_of(metric).calculate(&xd, &yd, false)
    });
    match r {
        Err(_) => (6, 0.0),
        Ok(Ok(v)) => (0, v.get_value()),
        Ok(Err(DistanceError::StorageMismatch)) => (1, 0.0),
        Ok(Err(DistanceError::CalculationError)) => (2, 0.0),
    }
}

#[test]
fn dump_hot_path_fixtures() {
    let dir = PathBuf::from(std::env::var("CDB_FIXTURE_DIR").expect("set CDB_FIXTURE_DIR"));
    std::fs::create_dir_all(&dir).unwrap();
    std::panic::set_hook(Box::new(|_| {})); // unimplemented!() arms are recorded, not printed
    let mut out = Out { f: File::create(dir.join("hotpath_ref_v1.cdbf")).unwrap() };
    let q8 = ScalarQuantization;

    for &dim in &[8usize, 31, 32, 33, 128, 768, 1024] {
        let (m, q) = corpus_for(dim);
        let (n, nq) = (m.len(), q.len());
        let flat = |v: &Vec<Vec<f32>>| v.iter().flatten().copied().collect::<Vec<f32>>();
        out.f32s(&format!("d{dim}/corpus"), &[n as u64, dim as u64], &flat(&m));
        out.f32s(&format!("d{dim}/queries"), &[nq as u64, dim as u64], &flat(&q));
        // dot_product_f32 (AVX2+FMA path on x86_64) and the sequential magnitudes finalize_ann_results uses
        let mut dots = Vec::new();
        for qv in &q {
            for row in &m {
                dots.push(dot_product_f32(qv, row));
            }
        }
        out.f32s(&format!("d{dim}/f32_dot"), &[nq as u64, n as u64], &dots);
        let mags: Vec<f32> = m.iter().map(|r| r.iter().map(|x| x * x).sum::<f32>().sqrt()).collect();
        let qmags: Vec<f32> = q.iter().map(|r| r.iter().map(|x| x * x).sum::<f32>().sqrt()).collect();
        out.f32s(&format!("d{dim}/f32_mag"), &[n as u64], &mags);
        out.f32s(&format!("d{dim}/f32_qmag"), &[nq as u64], &qmags);

        for st in 0u32..6 {
            let qs = |v: &Vec<f32>| q8.quantize(v, storage_type(st), (-1.0, 1.0)).unwrap();
            let rows: Vec<Storage> = m.iter().map(qs).collect();
            let qrows: Vec<Storage> = q.iter().map(qs).collect();
            let cb = code_bytes(&rows[0]).len() as u64;
            out.u8s(&format!("d{dim}/st{st}/codes"), &[n as u64, cb], &rows.iter().flat_map(code_bytes).collect::<Vec<u8>>());
            out.f32s(&format!("d{dim}/st{st}/mag"), &[n as u64], &rows.iter().map(mag_of).collect::<Vec<f32>>());
            out.u8s(&format!("d{dim}/st{st}/qcodes"), &[nq as u64, cb], &qrows.iter().flat_map(code_bytes).collect::<Vec<u8>>());
            out.f32s(&format!("d{dim}/st{st}/qmag"), &[nq as u64], &qrows.iter().map(mag_of).collect::<Vec<f32>>());
            // raw dot products of the storage type (before the metric's formula)
            let mut raw = Vec::new();
            for x in &qrows {
                for y in &rows {
                    raw.push(match (x, y) {
                        (Storage::UnsignedByte { quant_vec: a, .. }, Storage::UnsignedByte { quant_vec: b, .. }) => dot_product_u8(a, b) as f32,
                        (Storage::SubByte { quant_vec: a, resolution: 1, .. }, Storage::SubByte { quant_vec: b, .. }) => dot_product_binary(a, b, 1),
                        (Storage::SubByte { quant_vec: a, resolution: 2, .. }, Storage::SubByte { quant_vec: b, .. }) => dot_product_quaternary(a, b, 2),
                        (Storage::SubByte { quant_vec: a, resolution: 3, .. }, Storage::SubByte { quant_vec: b, .. }) => dot_product_octal(a, b, 3),
                        (Storage::HalfPrecisionFP { quant_vec: a, .. }, Storage::HalfPrecisionFP { quant_vec: b, .. }) => dot_product_f16(a, b),
                        (Storage::FullPrecisionFP { vec: a, .. }, Storage::FullPrecisionFP { vec: b, .. }) => dot_product_f32(a, b),
                        _ => f32::NAN,
                    });
                }
            }
            out.f32s(&format!("d{dim}/st{st}/dot"), &[nq as u64, n as u64], &raw);
            for metric in 0u32..4 {
                let (mut val, mut status) = (Vec::new(), Vec::new());
                for x in &qrows {
                    for y in &rows {
                        let (s, v) = calc(metric, x, y);
                        status.push(s);
                        val.push(v);
                    }
                }
                out.f32s(&format!("d{dim}/st{st}/m{metric}/value"), &[nq as u64, n as u64], &val);
                out.i8s(&format!("d{dim}/st{st}/m{metric}/status"), &[nq as u64, n as u64], &status);
            }
        }
        // u8 with a non-default values_range (clamp + scale arm of scalar.rs:17-24)
        let rows: Vec<Storage> = m.iter().map(|v| q8.quantize(v, StorageType::UnsignedByte, (-0.5, 0.75)).unwrap()).collect();
        out.u8s(&format!("d{dim}/st0_range/codes"), &[n as u64, dim as u64], &rows.iter().flat_map(code_bytes).collect::<Vec<u8>>());
        out.f32s(&format!("d{dim}/st0_range/mag"), &[n as u64], &rows.iter().map(mag_of).collect::<Vec<f32>>());
    }

    // ---- replica-kind arms of CosineSimilarity::calculate (cosine.rs:34-102): f16 storage, D = 16, 5 metadata dims
    {
        let mv = synth_matrix(0x3D7A, 2, 16);
        let sx = q8.quantize(&mv[0], StorageType::HalfPrecisionFP, (-1.0, 1.0)).unwrap();
        let sy = q8.quantize(&mv[1], StorageType::HalfPrecisionFP, (-1.0, 1.0)).unwrap();
        let pat_a = vec![1i32, 0, 1, 1, 0];
        let pat_b = vec![0i32, 1, 1, 0, 0];
        let zeros = vec![0i32; 5];
        let mag = |b: &Vec<i32>| (b.iter().map(|x| (x * x) as f32).sum::<f32>()).sqrt();
        let sides: Vec<(Option<u32>, Option<Vec<i32>>)> = vec![
            (None, None), (None, Some(pat_a.clone())), (Some(5), Some(zeros)), (Some(8), Some(pat_a.clone())),
            (Some(9), Some(pat_b.clone())), (Some(u32::MAX - 257), Some(pat_a.clone())), (Some(u32::MAX - 2), Some(pat_b)),
            (Some(u32::MAX - 258), Some(pat_a.clone())), (Some(u32::MAX), Some(pat_a)),
        ];
        let mut table = Vec::new();
        for (xid, xb) in &sides {
            for (yid, yb) in &sides {
                let xi = xid.map(InternalId::from);
                let yi = yid.map(InternalId::from);
                let xm = xb.as_ref().map(|b| Metadata { mag: mag(b), mbits: b.clone() });
                let ym = yb.as_ref().map(|b| Metadata { mag: mag(b), mbits: b.clone() });
                let r = std::panic::catch_unwind(|| {
                    let xd = VectorData { id: xi.as_ref(), quantized_vec: &sx, metadata: xm.as_ref() };
                    let yd = VectorData { id: yi.as_ref(), quantized_vec: &sy, metadata: ym.as_ref() };
                    DistanceMetric::Cosine.calculate(&xd, &yd, false)
                });
                let (s, v) = match r {
                    Err(_) => (7u32, 0.0f32), // unreachable!() arm
                    Ok(Ok(v)) => (0, v.get_value()),
                    Ok(Err(DistanceError::StorageMismatch)) => (1, 0.0),
                    Ok(Err(DistanceError::CalculationError)) => (2, 0.0),
                };
                table.push(s);
                table.push(v.to_bits());
            }
        }
        out.u32s("metadata/arm_table", &[sides.len() as u64, sides.len() as u64, 2], &table);
    }

    // ---- PerformantFixedSet (fixedset.rs): lossy membership after a fixed insert sequence
    {
        let mut members = Vec::new();
        for &len in &[16usize, 32, 64] {
            let mut fs = PerformantFixedSet::new(len);
            let ids: Vec<u32> = (0..200u64).map(|i| (synth_value(0xF1ED, i).to_bits() >> 3) % 100_000).collect();
            for id in &ids[..100] {
                fs.insert(*id);
            }
            for id in &ids {
                members.push(fs.is_member(*id) as u8);
            }
        }
        out.u8s("fixedset/is_member", &[3, 200], &members);
    }

    // ---- prop.data: node property file written by the reference's own serializer
    {
        let path = dir.join("prop.data");
        let _ = std::fs::remove_file(&path);
        let mut f = OpenOptions::new().read(true).write(true).create(true).open(&path).unwrap();
        let (m, _) = corpus_for(32);
        let mut locs = Vec::new();
        for (i, row) in m.iter().enumerate() {
            let s = q8.quantize(row, StorageType::UnsignedByte, (-1.0, 1.0)).unwrap();
            let (off, len) = write_prop_value_to_file(&InternalId::from(i as u32 * 3 + 1), &s, &mut f).unwrap();
            locs.push(off.0);
            locs.push(len.0);
            if i % 4 == 1 {
                // collections with a metadata schema interleave replica Metadata records in the same file
                let md = Arc::new(Metadata { mag: 2.0f32.sqrt(), mbits: vec![1, 0, 1, 0, 0] });
                let (off, len) = write_prop_metadata_to_file(InternalId::from(1000 + i as u32), md, &mut f).unwrap();
                locs.push(off.0);
                locs.push(len.0);
            }
        }
        f.flush().unwrap();
        out.u32s("prop/locations", &[(locs.len() / 2) as u64, 2], &locs);
    }

    // ---- itoe.dim / itoe.<version>.data: TreeMap<InternalId, RawVectorEmbedding> as Collection::new builds it
    {
        let _ = std::fs::remove_file(dir.join("itoe.dim"));
        let dim_file = OpenOptions::new().read(true).write(true).truncate(false).create(true).open(dir.join("itoe.dim")).unwrap();
        let dim_bufman = BufferManager::new(dim_file, 8192).unwrap();
        let root: Arc<std::path::Path> = dir.clone().into();
        let data_bufmans = BufferManagerFactory::new(root, |root, version: &VersionNumber| root.join(format!("itoe.{}.data", **version)), 8192);
        let map: TreeMap<InternalId, RawVectorEmbedding> = TreeMap::new(dim_bufman, data_bufmans);
        let (m, _) = corpus_for(32);
        for (i, row) in m.iter().enumerate() {
            let emb = RawVectorEmbedding {
                id: VectorId::from(format!("vec-{i}")),
                document_id: None,
                dense_values: Some(row.clone()),
                metadata: None,
                sparse_values: None,
                text: None,
            };
            map.insert(VersionNumber::from(0), &InternalId::from(i as u32 * 3 + 1), emb);
        }
        // newest state wins: overwrite one key in a later version, delete another
        let emb = RawVectorEmbedding {
            id: VectorId::from("vec-2-v1".to_string()),
            document_id: None,
            dense_values: Some(m[5].clone()),
            metadata: None,
            sparse_values: None,
            text: None,
        };
        map.insert(VersionNumber::from(1), &InternalId::from(2 * 3 + 1), emb);
        map.delete(VersionNumber::from(1), &InternalId::from(4 * 3 + 1));
        map.serialize().unwrap();
    }
    let _ = std::panic::take_hook();
    println!("fixtures written to {}", dir.display());
}

// ---------------------------------------------------------------- TF-IDF index files
// tests/tfidf_files.py::reference_fixture_script restates this script; keep the two identical.
fn tfidf_hashes() -> Vec<u32> {
    let mut h = Vec::new();
    for dim in [0u32, 1, 5, 21, 4096, 65535] {
        for q in [0u32, 1, 2, 3, 4, 5, 0x7FFF, 0xFFFF] {
            h.push(q << 16 | dim);
        }
    }
    h
}

fn tfidf_doc(doc: u32, hashes: &[u32]) -> Vec<(u32, f32)> {
    let mut pairs = Vec::new();
    for (j, &h) in hashes.iter().enumerate() {
        if (doc as usize + j) % 3 == 0 {
            let tf = if (doc as usize + j) % 7 == 0 { -0.0f32 } else { ((doc as usize * 7 + j) % 13) as f32 * 0.25 };
            pairs.push((h, tf));
        }
    }
    pairs
}

#[test]
fn dump_tfidf_fixtures() {
    let dir = PathBuf::from(std::env::var("CDB_FIXTURE_DIR").expect("set CDB_FIXTURE_DIR")).join("tf_idf_index");
    let _ = std::fs::remove_dir_all(&dir);
    std::fs::create_dir_all(&dir).unwrap();
    let work = std::env::temp_dir().join(format!("cdb_tfidf_fixture_{}", std::process::id()));
    let _ = std::fs::remove_dir_all(&work);
    std::fs::create_dir_all(&work).unwrap();
    let hashes = tfidf_hashes();
    let root = TFIDFIndexRoot::new(work.clone()).unwrap();
    // (version, first document, end document, deleted documents): each version inserts, then deletes, then serializes
    let script: [(u32, u32, u32, &[u32]); 3] = [(1, 0, 8, &[2]), (2, 8, 14, &[4, 9]), (3, 14, 18, &[10, 15, 0])];
    for (v, d0, d1, deletes) in script {
        let version = VersionNumber::from(v);
        for doc in d0..d1 {
            for (h, tf) in tfidf_doc(doc, &hashes) {
                root.insert(h, tf, doc, version).unwrap();
            }
            root.total_documents_count.fetch_add(1, std::sync::atomic::Ordering::Relaxed);
        }
        for &doc in deletes {
            for (h, _) in tfidf_doc(doc, &hashes) {
                root.delete(h, doc, version).unwrap();
            }
            root.total_documents_count.fetch_sub(1, std::sync::atomic::Ordering::Relaxed);
        }
        root.serialize().unwrap();
        root.cache.flush_all().unwrap();
    }
    drop(root);
    for entry in std::fs::read_dir(&work).unwrap() {
        let p = entry.unwrap().path();
        std::fs::copy(&p, dir.join(p.file_name().unwrap())).unwrap();
    }
    let _ = std::fs::remove_dir_all(&work);
    println!("tf_idf_index fixtures written to {}", dir.display());
}
